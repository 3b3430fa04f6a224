// lio.cu — LIO front-end hot path: fused k-NN + plane fit + point-to-plane residual/Jacobian (K3+K4)
// with in-kernel J^T J / J^T r reduction (K5), degeneracy sums, map_incremental (K2), and the host
// driver of the iterated ESKF.
//
// Replaces (reference: slam/mapping/fastlio/src/laserMapping.cpp):
//   h_share_model_geometric :813-982   -> lio_hmodel_kernel (+ lio_degen_kernel for :934-980)
//   esti_plane  include/common_lib.h:236-268 -> esti_plane_dev (Householder QR with column
//                                          pivoting in fp32, as Eigen's ColPivHouseholderQR)
//   map_incremental :523-576            -> lio_map_incremental_kernel
//   fastlio_main per-scan body :1126-1387 -> lsd_lio_scan
// Reduction layout: the reference materialises h_x (N_eff x 15 doubles) and forms h_x^T h_x on the
// CPU (esekfom.hpp:1784).  Here every thread owns one Jacobian row in registers, the 21 unique
// entries of the non-zero 6x6 block + 6 entries of h_x^T h + sum|res| + count are reduced by warp
// shuffles, per-block partials go to HBM and the last block to finish folds them in a fixed order
// (bit-reproducible).  No N x 15 matrix ever exists.
#include <unistd.h>

#include <chrono>

#include "eskf.hpp"
#include "knn.cuh"
#include "lio.h"
#include "map.h"
#include "voxelgrid.h"

namespace lsd {

constexpr int kNV = 32;        // reduction slots per block (29 used + n)
constexpr int kLioBlock = 256;
constexpr int kLioMaxGrid = 2 * kNumSms;  // 2 blocks per SM: the final fold reads <= kLioMaxGrid x 32 partials

struct LioPose { double R[9], t[3], RL[9], tL[3]; };

// ---------------------------------------------------------------- esti_plane (common_lib.h:236-268)
// A (5x3) n = -1 by Householder QR with column pivoting in fp32, every sum in the order Eigen's ColPivHouseholderQR takes on the
// reference's x86-64 build (4-float packets, no FMA; -fmad=false here): a whole column as ((t0+t2)+(t1+t3))+t4, a run-time
// tail of four as (t0+t2)+(t1+t3), shorter tails left to right, the upper-triangular solve column by column, |n|^2 as
// t0+(t1+t2).  The plane coefficients are bit-identical to the compiled reference's (oracle/lsd_oracle.c::orc_esti_plane is
// pinned to it on 1 M planes and states the rules with their Eigen sources).
__device__ __forceinline__ void swap_f(float& a, float& b) { float t = a; a = b; b = t; }
// sum of t[R0..4] in Eigen's run-time-size order
template <int R0>
__device__ __forceinline__ float red_tail(const float (&t)[5]) {
  if (R0 == 1) return (t[1] + t[3]) + (t[2] + t[4]);
  if (R0 == 2) return (t[2] + t[3]) + t[4];
  if (R0 == 3) return t[3] + t[4];
  return t[4];
}
template <int K>
__device__ __forceinline__ void esti_qr_step(float (&A)[5][3], float (&b)[5], float (&hc)[3], float (&nu)[3], float (&nd)[3], int (&perm)[3],
                                             int& nonzero, float th_helper, float downdate) {
  int big = K;
  float bn = nu[K];
#pragma unroll
  for (int j = K + 1; j < 3; j++) if (nu[j] > bn) { bn = nu[j]; big = j; }
  if (nonzero == 3 && bn * bn < th_helper * (float)(5 - K)) nonzero = K;
#pragma unroll
  for (int j = K + 1; j < 3; j++) {
    if (big == j) {
#pragma unroll
      for (int r = 0; r < 5; r++) swap_f(A[r][K], A[r][j]);
      swap_f(nu[K], nu[j]); swap_f(nd[K], nd[j]);
      int ti = perm[K]; perm[K] = perm[j]; perm[j] = ti;
    }
  }
  float t[5];
#pragma unroll
  for (int r = 0; r < 5; r++) t[r] = A[r][K] * A[r][K];
  const float tail = red_tail<K + 1>(t);
  const float c0 = A[K][K];
  float beta, tau;
  if (tail <= 1.17549435e-38f) {
    tau = 0.f; beta = c0;
#pragma unroll
    for (int r = K + 1; r < 5; r++) A[r][K] = 0.f;
  } else {
    beta = sqrtf(c0 * c0 + tail);
    if (c0 >= 0.f) beta = -beta;
    const float den = c0 - beta;
#pragma unroll
    for (int r = K + 1; r < 5; r++) A[r][K] = A[r][K] / den;
    tau = (beta - c0) / beta;
  }
  hc[K] = tau; A[K][K] = beta;
  if (tau != 0.f) {
#pragma unroll
    for (int j = K + 1; j < 3; j++) {
#pragma unroll
      for (int r = 0; r < 5; r++) t[r] = A[r][K] * A[r][j];
      float tmp = red_tail<K + 1>(t);
      tmp += A[K][j];
      A[K][j] -= tau * tmp;
#pragma unroll
      for (int r = K + 1; r < 5; r++) A[r][j] -= (tau * A[r][K]) * tmp;
    }
  }
#pragma unroll
  for (int j = K + 1; j < 3; j++) {
    if (nu[j] != 0.f) {
      float q = fabsf(A[K][j]) / nu[j];
      q = (1.f + q) * (1.f - q);
      if (q < 0.f) q = 0.f;
      const float rr = nu[j] / nd[j];
      const float t2 = q * (rr * rr);
      if (t2 <= downdate) {
#pragma unroll
        for (int r = 0; r < 5; r++) t[r] = A[r][j] * A[r][j];
        nd[j] = sqrtf(red_tail<K + 1>(t)); nu[j] = nd[j];
      } else {
        nu[j] *= sqrtf(q);
      }
    }
  }
}
template <int K>
__device__ __forceinline__ void esti_apply_b(const float (&A)[5][3], float (&b)[5], const float (&hc)[3], int nonzero) {
  if (K < nonzero && hc[K] != 0.f) {
    float t[5];
#pragma unroll
    for (int r = 0; r < 5; r++) t[r] = A[r][K] * b[r];
    float tmp = red_tail<K + 1>(t);
    tmp += b[K];
    b[K] -= hc[K] * tmp;
#pragma unroll
    for (int r = K + 1; r < 5; r++) b[r] -= (hc[K] * A[r][K]) * tmp;
  }
}
__device__ __forceinline__ bool esti_plane_dev(const float (&px)[5], const float (&py)[5], const float (&pz)[5], float thr,
                                               float (&pabcd)[4]) {
  const float FEPS = 1.1920929e-07f;
  float A[5][3], b[5];
#pragma unroll
  for (int r = 0; r < 5; r++) { A[r][0] = px[r]; A[r][1] = py[r]; A[r][2] = pz[r]; b[r] = -1.0f; }
  float hc[3], nu[3], nd[3];
  int perm[3] = {0, 1, 2};
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float t0 = A[0][k] * A[0][k], t1 = A[1][k] * A[1][k], t2 = A[2][k] * A[2][k], t3 = A[3][k] * A[3][k], t4 = A[4][k] * A[4][k];
    nu[k] = nd[k] = sqrtf(((t0 + t2) + (t1 + t3)) + t4);
  }
  float mxn = nu[0];
  if (nu[1] > mxn) mxn = nu[1];
  if (nu[2] > mxn) mxn = nu[2];
  const float th_helper = (mxn * FEPS) * (mxn * FEPS) / 5.0f;
  const float downdate = sqrtf(FEPS);
  int nonzero = 3;
  esti_qr_step<0>(A, b, hc, nu, nd, perm, nonzero, th_helper, downdate);
  esti_qr_step<1>(A, b, hc, nu, nd, perm, nonzero, th_helper, downdate);
  esti_qr_step<2>(A, b, hc, nu, nd, perm, nonzero, th_helper, downdate);
  float x[3] = {0.f, 0.f, 0.f};
  if (nonzero > 0) {
    esti_apply_b<0>(A, b, hc, nonzero);
    esti_apply_b<1>(A, b, hc, nonzero);
    esti_apply_b<2>(A, b, hc, nonzero);
    // upper-triangular solve, column by column from the last (Eigen's triangular_solve_vector, ColMajor)
#pragma unroll
    for (int i = 2; i >= 0; i--) {
      if (i < nonzero && b[i] != 0.f) {
        b[i] /= A[i][i];
#pragma unroll
        for (int r = 0; r < i; r++) b[r] -= b[i] * A[r][i];
      }
    }
#pragma unroll
    for (int i = 0; i < 3; i++) {
      if (i < nonzero) {
        if (perm[i] == 0) x[0] = b[i]; else if (perm[i] == 1) x[1] = b[i]; else x[2] = b[i];
      }
    }
  }
  const float n = sqrtf(x[0] * x[0] + (x[1] * x[1] + x[2] * x[2]));
  pabcd[0] = x[0] / n; pabcd[1] = x[1] / n; pabcd[2] = x[2] / n; pabcd[3] = (float)(1.0 / (double)n);
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const float v = pabcd[0] * px[j] + pabcd[1] * py[j] + pabcd[2] * pz[j] + pabcd[3];
    if (fabs((double)v) > (double)thr) ok = false;
  }
  return ok;
}

// ---------------------------------------------------------------- grid reduction
// Result buffer layout (doubles): [0..20] upper triangle of the 6x6 h_x^T h_x, [21..26] h_x^T h,
// [27] sum |res|, [28] n_eff, [29] feats_down_size, [48..53] degeneracy sums.
constexpr int kResDegen = 48, kResWaitCycles = 56, kResSeq = 62, kResSeqDegen = 63, kResDoubles = 64;

// symmetric 3x3 eigen-decomposition (cyclic Jacobi); V columns = eigenvectors.  Stands in for
// Eigen::SelfAdjointEigenSolver at laserMapping.cpp:941; only |v . n| and V diag(mask) V^T are used,
// both independent of eigenvector sign and order.
static void eig3_sym(const double* Ain, double* V, double* w) {
  double A[9];
  for (int i = 0; i < 9; i++) { A[i] = Ain[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 60; sweep++) {
    if (fabs(A[1]) + fabs(A[2]) + fabs(A[5]) <= 1e-18 * (fabs(A[0]) + fabs(A[4]) + fabs(A[8]))) break;
    for (int p = 0; p < 2; p++) for (int q = p + 1; q < 3; q++) {
      const double apq = A[3 * p + q];
      if (fabs(apq) < 1e-300) continue;
      const double th = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
      const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
      for (int k = 0; k < 3; k++) { double x = A[3 * k + p], y = A[3 * k + q]; A[3 * k + p] = c * x - sn * y; A[3 * k + q] = sn * x + c * y; }
      for (int k = 0; k < 3; k++) { double x = A[3 * p + k], y = A[3 * q + k]; A[3 * p + k] = c * x - sn * y; A[3 * q + k] = sn * x + c * y; }
      for (int k = 0; k < 3; k++) { double x = V[3 * k + p], y = V[3 * k + q]; V[3 * k + p] = c * x - sn * y; V[3 * k + q] = sn * x + c * y; }
    }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
}

// Called by every thread of every block after the block has written partials[blockIdx][0..NV).
// The last block to arrive folds all partials in a fixed order (slices of blocks, ascending) into
// result[0..NV) — bit-reproducible for a given grid size.
// `result` is HOST memory mapped into the device address space: the last block publishes the sums
// and then a sequence number the host spins on (no cudaMemcpy, no stream synchronise per iteration).
template <int NV>
__device__ __forceinline__ void grid_finalize(double* __restrict__ partials, unsigned* __restrict__ done,
                                              volatile double* __restrict__ result, int res_off, int n_extra_slot, double extra,
                                              int seq_slot, double seq, const ShardComm& sc, int inbox_region) {
  __shared__ double sm_fin[8][kNV];
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int slices = blockDim.x >> 5;
  const int j = threadIdx.x & 31, slice = threadIdx.x >> 5;
  double s = 0.0;
  if (j < NV) {  // ascending block order per slice, 8 independent loads in flight
    const int G = (int)gridDim.x;
    int b = slice;
    for (; b + 7 * slices < G; b += 8 * slices) {
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; u++) v[u] = __ldcg(partials + (size_t)(b + u * slices) * kNV + j);
#pragma unroll
      for (int u = 0; u < 8; u++) s += v[u];
    }
    for (; b < G; b += slices) s += __ldcg(partials + (size_t)b * kNV + j);
  }
  sm_fin[slice][j] = s;
  __syncthreads();
  if (threadIdx.x < NV) {
    double t = 0.0;
    for (int w = 0; w < slices; w++) t += sm_fin[w][threadIdx.x];
    sm_fin[0][threadIdx.x] = t;
  }
  __syncthreads();
  if (sc.world > 1) {
    // Cross-rank all-reduce fused into the reduction kernel: the last block stores this rank's totals
    // into every rank's inbox over NVLink, publishes a sequence number, waits for the other ranks'
    // and folds the world's contributions in rank order (deterministic).  No NCCL call, no extra launch.
    const long long iseq = (long long)seq;
    const long long t_x0 = clock64();   // exchange time (stores + peers' arrival), published in result[kResWaitCycles]
    const size_t base = (size_t)inbox_region * kInboxRegion + (size_t)((iseq & 1) * kMaxRanks) * kInboxSlot;
    if (threadIdx.x < NV) {
      const double v = sm_fin[0][threadIdx.x];
      for (int p = 0; p < sc.world; p++) sc.inbox[p][base + (size_t)sc.rank * kInboxSlot + threadIdx.x] = v;
      __threadfence_system();
    }
    __syncthreads();
    if (threadIdx.x < sc.world) {
      volatile double* flag = sc.inbox[threadIdx.x] + base + (size_t)sc.rank * kInboxSlot + (kInboxSlot - 1);
      *flag = seq;
      __threadfence_system();
      volatile double* mine = sc.inbox[sc.rank] + base + (size_t)threadIdx.x * kInboxSlot + (kInboxSlot - 1);
      while (*mine != seq) {}
    }
    __syncthreads();
    __threadfence_system();
    if (threadIdx.x < NV) {
      double t = 0.0;
      for (int r = 0; r < sc.world; r++) t += *(volatile double*)(sc.inbox[sc.rank] + base + (size_t)r * kInboxSlot + threadIdx.x);
      sm_fin[0][threadIdx.x] = t;
    }
    if (threadIdx.x == 0 && inbox_region == 0) result[kResWaitCycles] = (double)(clock64() - t_x0);
    __syncthreads();
  }
  // One system-scope fence round: every writer fences its own stores, the barrier makes them happen-before thread 0's
  // sequence-number store (fence cumulativity), so the host that sees `seq` sees the sums.  (A second fence in thread 0 cost
  // another PCIe round trip per evaluation.)
  if (threadIdx.x < NV) result[res_off + threadIdx.x] = sm_fin[0][threadIdx.x];
  if (threadIdx.x == NV && n_extra_slot >= 0) result[n_extra_slot] = extra;
  if (threadIdx.x == NV + 1) *done = 0u;
  if (threadIdx.x <= NV + 1) __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) result[seq_slot] = seq;  // published last
}

// thread-per-item kernels: warp-shuffle reduce vals[NV] into partials[block]
template <int NV>
__device__ __forceinline__ void block_partials(double (&vals)[NV], double* __restrict__ partials) {
  __shared__ double sm_bp[8][kNV];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if constexpr (NV > 8) {
    const double v = warp_sum_to_lane<NV>(vals);   // lane j <- warp total of vals[j], same bits as warp_sum
    if (lane < NV) sm_bp[warp][lane] = v;
  } else {
#pragma unroll
    for (int j = 0; j < NV; j++) {
      const double v = warp_sum(vals[j]);
      if (lane == 0) sm_bp[warp][j] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sm_bp[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kNV + threadIdx.x] = s;
  }
}

// Jacobian row (laserMapping.cpp:903-932, extrinsic_est_en == false) and residual for one point
struct RowH { double row[6]; double h; };
__device__ __forceinline__ RowH make_row(const LioPose& ps, double lx, double ly, double lz, const float (&pabcd)[4], float pd2) {
  RowH r;
  const double nx = pabcd[0], ny = pabcd[1], nz = pabcd[2];
  const double cx = ps.R[0] * nx + ps.R[3] * ny + ps.R[6] * nz;  // R^T n
  const double cy = ps.R[1] * nx + ps.R[4] * ny + ps.R[7] * nz;
  const double cz = ps.R[2] * nx + ps.R[5] * ny + ps.R[8] * nz;
  r.row[0] = nx; r.row[1] = ny; r.row[2] = nz;
  r.row[3] = ly * cz - lz * cy; r.row[4] = lz * cx - lx * cz; r.row[5] = lx * cy - ly * cx;
  r.h = -(double)pd2;
  return r;
}

__constant__ unsigned char c_tri[21][2] = {{0,0},{0,1},{0,2},{0,3},{0,4},{0,5},{1,1},{1,2},{1,3},{1,4},{1,5},{2,2},{2,3},{2,4},{2,5},
                                           {3,3},{3,4},{3,5},{4,4},{4,5},{5,5}};

// ---------------------------------------------------------------- the reference's neighbour ORDER (lsd_lio_set_reference_order)
// IVox::GetClosestPoint leaves its (up to) five neighbours in the order std::nth_element's introselect produces on the
// candidate sequence (ivox3d.h:159-164; per voxel with more than five in range: ivox3d_node.hpp:118-123), and esti_plane's
// fp32 solve depends on the row order.  With the switch on, the search keeps EVERY in-range candidate of a query, puts them in
// the reference's sequence (stencil cell in nearby_grids_ order, then insertion order = ascending id) and replays libstdc++'s
// algorithm on the distances (DistPoint::operator< compares nothing else): warp_nth_element below for up to 32 candidates — the
// case that matters: 11 on average, 29 at most on the benchmark map — and rs_reference_order, the algorithm as written, run by
// lane 0 on shared memory, for longer sequences (NEARBY74 in the first second of a run, crowded maps) and where introselect
// would leave for __heap_select.  oracle/lsd_oracle.c::ref_nth_element states the algorithm with its libstdc++ sources and is
// pinned id for id to the compiled iVox.  A query whose candidates overflow the search's list (kCandCap = 256) is answered in
// the canonical (d2, id) order and counted (lsd_lio_reference_order_fallbacks).
//
// Where the replay runs: one thread per query inside the plane-fit kernel takes that kernel's registers, and a kernel of its
// own is a chain of ~3 k dependent instructions per thread with nothing to hide latency behind; the search's own warp,
// below, keeps the lanes busy.  Gathering cell by cell (warp prefix sum of per-cell counts) so that the list is the sequence
// without the all-pairs placement needs seven distances and ids per lane held in registers.
#ifdef LSD_SIMT_EMU
#define RS_INL __device__
#define RS_ONE __device__
#else
#define RS_INL __device__ __forceinline__
#define RS_ONE __device__ __noinline__   // rs_nth_element: ONE copy (it has three call sites); everything inside it is inlined
#endif
RS_INL void rs_swap(unsigned char* r, unsigned char* ix, int a, int b) {
  const unsigned char t = r[a]; r[a] = r[b]; r[b] = t;
  const unsigned char u = ix[a]; ix[a] = ix[b]; ix[b] = u;
}
RS_INL void rs_adjust_heap(unsigned char* r, unsigned char* ix, int first, int hole, int len, unsigned char vr, unsigned char vi) {   // std::__adjust_heap + __push_heap
  const int top = hole;
  int child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (r[first + child] < r[first + child - 1]) child--;
    r[first + hole] = r[first + child]; ix[first + hole] = ix[first + child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    r[first + hole] = r[first + child - 1]; ix[first + hole] = ix[first + child - 1];
    hole = child - 1;
  }
  int parent = (hole - 1) / 2;
  while (hole > top && r[first + parent] < vr) {
    r[first + hole] = r[first + parent]; ix[first + hole] = ix[first + parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  r[first + hole] = vr; ix[first + hole] = vi;
}
// std::nth_element(first, nth, last) of libstdc++ on positions of the sequence (bits/stl_algo.h __introselect)
RS_INL void rs_nth_element_impl(unsigned char* r, unsigned char* ix, int first, int nth, int last) {
  if (first == last || nth == last) return;
  int depth = 0;
  for (int n = last - first; n > 1; n >>= 1) depth++;
  depth *= 2;
  while (last - first > 3) {
    if (depth == 0) {   // __heap_select(first, nth + 1, last) + iter_swap(first, nth)
      const int middle = nth + 1, len = middle - first;
      if (len >= 2)
        for (int parent = (len - 2) / 2;; parent--) {
          rs_adjust_heap(r, ix, first, parent, len, r[first + parent], ix[first + parent]);
          if (parent == 0) break;
        }
      for (int i = middle; i < last; i++)
        if (r[i] < r[first]) {
          const unsigned char vr = r[i], vi = ix[i];
          r[i] = r[first]; ix[i] = ix[first];
          rs_adjust_heap(r, ix, first, 0, len, vr, vi);
        }
      rs_swap(r, ix, first, nth);
      return;
    }
    depth--;
    const int a = first + 1, b = first + (last - first) / 2, c = last - 1;   // __move_median_to_first
    const unsigned char ra = r[a], rb = r[b], rc_ = r[c];
    int med;
    if (ra < rb) med = rb < rc_ ? b : (ra < rc_ ? c : a);
    else med = ra < rc_ ? a : (rb < rc_ ? c : b);
    rs_swap(r, ix, first, med);
    int lo = first + 1, hi = last;                                         // __unguarded_partition
    const unsigned char pv = r[first];
    for (;;) {
      while (r[lo] < pv) lo++;
      hi--;
      while (pv < r[hi]) hi--;
      if (!(lo < hi)) break;
      rs_swap(r, ix, lo, hi);
      lo++;
    }
    if (lo <= nth) first = lo; else last = lo;
  }
  for (int i = first + 1; i < last; i++) {                                  // __insertion_sort
    const unsigned char vr = r[i], vi = ix[i];
    int j = i;
    if (vr < r[first]) {
      for (; j > first; j--) { r[j] = r[j - 1]; ix[j] = ix[j - 1]; }
    } else {
      while (vr < r[j - 1]) { r[j] = r[j - 1]; ix[j] = ix[j - 1]; j--; }
    }
    r[j] = vr; ix[j] = vi;
  }
}
RS_ONE void rs_nth_element(unsigned char* r, unsigned char* ix, int first, int nth, int last) { rs_nth_element_impl(r, ix, first, nth, last); }
// GetClosestPoint's ordering, serially, on a query's candidates in the reference's sequence (ck[t] = cell << 8 | rank of the
// distance): per-voxel truncation, the two nth_element calls.  Returns how many neighbours the reference returns (<= 5); their
// positions in the sequence are ix[0 ..).  Run by lane 0 of the search's warp for the queries warp_nth_element does not take.
RS_INL int rs_reference_order(unsigned char* r, unsigned char* ix, const unsigned short* __restrict__ ck, int n) {
  int m = 0;
  for (int a = 0; a < n;) {
    const unsigned short ca = ck[a];
    const int old = m;
    r[m] = (unsigned char)(ca & 0xff); ix[m] = (unsigned char)a; m++;
    int b = a + 1;
    for (; b < n; b++) {
      const unsigned short cb = ck[b];
      if ((cb >> 8) != (ca >> 8)) break;
      r[m] = (unsigned char)(cb & 0xff); ix[m] = (unsigned char)b; m++;
    }
    if (m - old > 5) {                                                      // KNNPointByCondition, K = 5 (crowded voxels: rare)
      rs_nth_element(r, ix, old, old + 4, m); m = old + 5;
    }
    a = b;
  }
#pragma unroll 1
  for (int c = 0; c < 2; c++) {                                             // ivox3d.h:159-164: nth_element(.., begin + 4, ..) if more than five, then (.., begin, ..)
    if (c == 0 && m <= 5) continue;
    if (m == 0) break;
    rs_nth_element(r, ix, 0, c == 0 ? 4 : 0, m);
    if (c == 0) m = 5;
  }
  return m;
}

// ---- the same replay, by the WARP that ran the search, for sequences of up to 32 candidates with no crowded voxel ------------
// Position p of the working sequence lives in lane p: key = fp32 bits of the distance, src = index into the search's list.
// A Hoare partition becomes two ballots (where the left / the right scan would stop) and a walk over their bits; its swaps are
// disjoint, so one shuffle per register applies them all.  No divergence, no memory: ~60 warp instructions per partition
// against ~3 k dependent per-thread instructions of the serial replay.  Returns false where libstdc++ would fall into
// __heap_select (depth limit): the serial replay then takes the query.
__device__ __forceinline__ bool warp_nth_element(unsigned& key, int& src, int first, int nth, int last) {
  const int lane = threadIdx.x & 31;
  if (first == last || nth == last) return true;
  int depth = 2 * (31 - __clz(last - first));                                  // 2 * std::__lg(last - first)
  while (last - first > 3) {
    if (depth == 0) return false;
    depth--;
    const int a = first + 1, b = first + (last - first) / 2, c = last - 1;     // __move_median_to_first(first, a, b, c)
    const unsigned ka = __shfl_sync(kFull, key, a), kb = __shfl_sync(kFull, key, b), kc = __shfl_sync(kFull, key, c);
    const int med = ka < kb ? (kb < kc ? b : (ka < kc ? c : a)) : (ka < kc ? a : (kb < kc ? c : b));
    {
      const int sl = lane == first ? med : (lane == med ? first : lane);
      key = __shfl_sync(kFull, key, sl); src = __shfl_sync(kFull, src, sl);
    }
    const unsigned pv = __shfl_sync(kFull, key, first);                       // __unguarded_partition(first + 1, last, first)
    const bool inr = lane > first && lane < last;
    unsigned mask_l = __ballot_sync(kFull, inr && !(key < pv));               // where "while (*lo < pivot) ++lo" stops
    unsigned mask_r = __ballot_sync(kFull, inr && !(pv < key)) | (1u << first);   // where "while (pivot < *hi) --hi" stops (the pivot itself at the latest)
    int lo = first + 1, hi = last, sl = lane;
    for (;;) {
      lo = __ffs((int)(mask_l & ~((1u << lo) - 1u))) - 1;
      hi--;
      hi = 31 - __clz((int)(mask_r & (hi >= 31 ? 0xffffffffu : ((2u << hi) - 1u))));
      if (!(lo < hi)) break;
      if (lane == lo) sl = hi; else if (lane == hi) sl = lo;                    // iter_swap(lo, hi), applied below
      mask_l |= 1u << hi; mask_r |= 1u << lo;                                   // what the swap put there stops the other scan
      lo++;
    }
    key = __shfl_sync(kFull, key, sl); src = __shfl_sync(kFull, src, sl);
    if (lo <= nth) first = lo; else last = lo;
  }
  // __insertion_sort(first, last): a stable sort of at most three elements
  const int cnt = last - first;
  if (cnt >= 2) {
    const unsigned k0 = __shfl_sync(kFull, key, first), k1 = __shfl_sync(kFull, key, first + 1);
    const unsigned k2 = cnt > 2 ? __shfl_sync(kFull, key, first + 2) : 0xffffffffu;
    const int r0 = (k1 < k0 ? 1 : 0) + (k2 < k0 ? 1 : 0);
    const int r1 = (k0 <= k1 ? 1 : 0) + (k2 < k1 ? 1 : 0);
    const int r2 = (k0 <= k2 ? 1 : 0) + (k1 <= k2 ? 1 : 0);
    int sl = lane;
    if (lane == first + r0) sl = first;
    if (lane == first + r1) sl = first + 1;
    if (cnt > 2 && lane == first + r2) sl = first + 2;
    key = __shfl_sync(kFull, key, sl); src = __shfl_sync(kFull, src, sl);
  }
  return true;
}

// ---------------------------------------------------------------- K3: neighbour search for the scan
// One warp per downsampled point (knn.cuh): body -> world, 5-NN in the hash-voxel map, neighbours
// written as Nearest_Points[i] (laserMapping.cpp:842-852).  Kept separate from the plane fit: the
// search wants one warp per query (19 probes in flight), the plane fit one thread per query.
constexpr int kHmWarps = 8;
__global__ void __launch_bounds__(kHmWarps * 32, 4) lio_knn_kernel(MapView mv, int stencil, const float4* __restrict__ body,
                                                                const int* __restrict__ n_ptr, int cap, LioPose ps,
                                                                float4* __restrict__ near, int* __restrict__ near_cnt,
                                                                int keep_stale, int* __restrict__ rows, int resize_parity,
                                                                int ref_order, unsigned* __restrict__ ref_fallbacks) {
  pdl_enter();
  __shared__ __align__(16) unsigned char s_list[kHmWarps * kWarpListBytes];
  __shared__ unsigned char s_cell[kHmWarps][kCandCap];
  __shared__ unsigned s_fkey[kHmWarps][32];
  __shared__ unsigned char s_fsrc[kHmWarps][32], s_fcell[kHmWarps][32];
  __shared__ unsigned short s_sck[kHmWarps][kCandCap];                                        // the serial replay's arrays
  __shared__ unsigned char s_sr[kHmWarps][kCandCap], s_six[kHmWarps][kCandCap], s_sp[kHmWarps][kCandCap];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = min(__ldcg(n_ptr), cap);
  if (resize_parity >= 0) {
    // Nearest_Points.resize(feats_down_size) (laserMapping.cpp:1273), folded into the scan's first search: rows the new
    // scan does not have are destroyed, so a later, larger scan finds them empty.  The reference returns before the
    // resize when feats_down_size < 5 (:1252-1256).  rows[2] is double-buffered by scan parity: this launch reads the
    // number of rows alive from rows[parity ^ 1] (published by the previous resize) and publishes its own in
    // rows[parity], so no block can read a value another block of the same launch has already replaced.
    const int prev = min(__ldcg(rows + (resize_parity ^ 1)), cap);
    if (n >= 5)
      for (int i = n + blockIdx.x * blockDim.x + threadIdx.x; i < prev; i += gridDim.x * blockDim.x) {
        near_cnt[i] = 0;
#pragma unroll
        for (int r = 0; r < 5; r++) near[(size_t)i * 5 + r] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
      }
    if (blockIdx.x == 0 && threadIdx.x == 0) rows[resize_parity] = n >= 5 ? n : prev;
  }
  WarpList wl = make_warp_list(s_list, warp);
  wl.cell = ref_order ? s_cell[warp] : nullptr;
  const LaneStencil ls = lane_stencil(stencil_slot(stencil));
  // (An L2-prefetch pass over the warp's queries was measured here and removed: +9 us per launch —
  // the kernel is bound by its dependent instruction chain per query, not by the cold HBM trip.)
  for (int i = blockIdx.x * kHmWarps + warp; i < n; i += gridDim.x * kHmWarps) {
    const float4 pb = __ldg(body + i);
    // body -> world in double (laserMapping.cpp:831-836), stored as fp32 like PointType
    const double bx = pb.x, by = pb.y, bz = pb.z;
    const double lx = ps.RL[0] * bx + ps.RL[1] * by + ps.RL[2] * bz + ps.tL[0];
    const double ly = ps.RL[3] * bx + ps.RL[4] * by + ps.RL[5] * bz + ps.tL[1];
    const double lz = ps.RL[6] * bx + ps.RL[7] * by + ps.RL[8] * bz + ps.tL[2];
    const float wx = (float)(ps.R[0] * lx + ps.R[1] * ly + ps.R[2] * lz + ps.t[0]);
    const float wy = (float)(ps.R[3] * lx + ps.R[4] * ly + ps.R[5] * lz + ps.t[1]);
    const float wz = (float)(ps.R[6] * lx + ps.R[7] * ly + ps.R[8] * lz + ps.t[2]);
    if (mv.shard_world > 1) {  // tile-sharded: only the owner of the query's home voxel resolves it
      const int3 hc = pos2grid(wx, wy, wz, mv.inv_res);
      if (!shard_owns(mv, hc.x, hc.y)) { if (lane == 0) near_cnt[i] = -1; continue; }
    }
    if (ref_order) {
      // every in-range candidate, then the reference's order on them: warp_nth_element for up to 32, the serial replay else
      knn_stencil_gather<5>(mv, ls, wx, wy, wz, 5.0f, wl);
      const int n = wl.n;
      if (n == 0) {                       // GetClosestPoint returns false before touching its output (ivox3d.h:155-157)
        if (!keep_stale) { if (lane == 0) near_cnt[i] = 0; if (lane < 5) near[(size_t)i * 5 + lane] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1)); }
        continue;
      }
      if (!wl.clipped) {
        int m = -1, src = 0;              // m >= 0: lanes j < m hold in `src` the list index of the j-th neighbour
        if (n <= 32) {
          // the reference's sequence: stencil cell in nearby_grids_ order, then the voxel's insertion order (= ascending id)
          const unsigned d = lane < n ? wl.d[lane] : 0xffffffffu;
          const int id = lane < n ? wl.id[lane] : 0x7fffffff;
          const int c = lane < n ? (int)wl.cell[lane] : 255;
          int pos = 0;
          for (int t = 0; t < n; t++) {
            const int ct = wl.cell[t]; const int it = wl.id[t];
            pos += (ct < c || (ct == c && it < id)) ? 1 : 0;
          }
          if (lane < n) { s_fkey[warp][pos] = d; s_fsrc[warp][pos] = (unsigned char)lane; s_fcell[warp][pos] = (unsigned char)c; }
          __syncwarp();
          unsigned key = lane < n ? s_fkey[warp][lane] : 0xffffffffu;
          src = lane < n ? (int)s_fsrc[warp][lane] : 0;
          int cellv = lane < n ? (int)s_fcell[warp][lane] : 256 + lane;
          __syncwarp();
          m = n;
          bool ok = true;
          for (;;) {     // KNNPointByCondition: a voxel with more than five candidates keeps nth_element's first five (ivox3d_node.hpp:118-123)
            const int prev = __shfl_up_sync(kFull, cellv, 1);
            const unsigned starts = __ballot_sync(kFull, lane < m && (lane == 0 || cellv != prev));
            const int start = 31 - __clz((int)(starts & (lane >= 31 ? 0xffffffffu : ((2u << lane) - 1u))));
            const unsigned above = lane >= 31 ? 0u : (starts & ~((2u << lane) - 1u));
            const int end = above ? __ffs((int)above) - 1 : m;
            const unsigned crowded = __ballot_sync(kFull, lane < m && lane == start && end - start > 5);
            if (!crowded) break;
            const int ra = __ffs((int)crowded) - 1;
            const int rb = __shfl_sync(kFull, end, ra);
            if (!warp_nth_element(key, src, ra, ra + 4, rb)) { ok = false; break; }
            const int drop = rb - (ra + 5);
            const int from = lane < ra + 5 ? lane : lane + drop;
            const unsigned k2 = __shfl_sync(kFull, key, from & 31); const int s2 = __shfl_sync(kFull, src, from & 31);
            const int c2 = __shfl_sync(kFull, cellv, from & 31);
            m -= drop;
            key = lane < m ? k2 : 0xffffffffu; src = s2; cellv = lane < m ? c2 : 256 + lane;
          }
          if (ok && m > 5) { ok = warp_nth_element(key, src, 0, 4, m); m = 5; }       // ivox3d.h:159-162
          if (ok) ok = warp_nth_element(key, src, 0, 0, m);                            // ivox3d.h:164
          if (!ok) m = -1;
        }
        if (m < 0) {
          // more than 32 candidates (NEARBY74, crowded maps) or introselect's depth limit: lane 0 replays libstdc++ serially
          unsigned short* ck = s_sck[warp]; unsigned char* sr = s_sr[warp]; unsigned char* six = s_six[warp]; unsigned char* sp = s_sp[warp];
          for (int p = lane; p < n; p += 32) {
            const unsigned d = wl.d[p]; const int id = wl.id[p]; const int c = wl.cell[p];
            int pos = 0, rk = 0;
            for (int t = 0; t < n; t++) {
              const int ct = wl.cell[t]; const int it = wl.id[t];
              pos += (ct < c || (ct == c && it < id)) ? 1 : 0;
              rk += wl.d[t] < d ? 1 : 0;
            }
            ck[pos] = (unsigned short)((c << 8) | rk); sp[pos] = (unsigned char)p;
          }
          __syncwarp();
          int mm = 0;
          if (lane == 0) mm = rs_reference_order(sr, six, ck, n);
          m = __shfl_sync(kFull, mm, 0);
          __syncwarp();
          src = lane < m ? (int)sp[six[lane]] : 0;
          __syncwarp();
        }
        float4 q = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
        if (lane < m) q = load_loc(mv, wl.loc[src]);
        if (lane < 5) near[(size_t)i * 5 + lane] = q;
        if (lane == 0) near_cnt[i] = m;
        __syncwarp();
        continue;
      }
      if (lane == 0) atomicAdd(ref_fallbacks, 1u);   // more candidates than the list holds: canonical order below
    }
    Neighbor nb;
    const int nf = knn_search_warp<5>(mv, stencil, ls, wx, wy, wz, 5.0f, wl, nb);
    // keep_stale: IVox::GetClosestPoint returns before clearing its output when nothing is in range (ivox3d.h:155-157)
    // and Nearest_Points outlives the scan (laserMapping.cpp:1273): row i then keeps what it held (lsd_lio_set_stale_rows)
    if (keep_stale && nf == 0) continue;
    float4 q = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
    if (lane < nf) q = load_loc(mv, nb.loc);
    if (lane < 5) near[(size_t)i * 5 + lane] = q;
    if (lane == 0) near_cnt[i] = nf;
  }
}

// ---------------------------------------------------------------- K4+K5: plane fit + residual/Jacobian + reduction
// One thread per downsampled point.  FIT: first evaluation after a search — fit the plane through
// Nearest_Points[i] and cache it; !FIT: iterations with ekfom_data.converge == false
// (laserMapping.cpp:842) keep Nearest_Points and the reference refits the same plane from the same
// 5 points, so the cached plane is exact.
template <bool FIT>
__global__ void __launch_bounds__(kLioBlock) lio_hmodel_kernel(const float4* __restrict__ body, const int* __restrict__ n_ptr,
                                                               int cap, LioPose ps, const float4* __restrict__ near,
                                                               const int* __restrict__ near_cnt, unsigned char* __restrict__ selected,
                                                               float4* __restrict__ pabcd_io, unsigned char* __restrict__ plane_ok,
                                                               float4* __restrict__ plane, float4* __restrict__ world,
                                                               double* __restrict__ partials, unsigned* __restrict__ done,
                                                               double* __restrict__ result, double seq, ShardComm sc) {
  pdl_enter();
  const int n_true = __ldcg(n_ptr);
  const int n = min(n_true, cap);
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 pb = __ldg(body + i);
    const double bx = pb.x, by = pb.y, bz = pb.z;
    const double lx = ps.RL[0] * bx + ps.RL[1] * by + ps.RL[2] * bz + ps.tL[0];
    const double ly = ps.RL[3] * bx + ps.RL[4] * by + ps.RL[5] * bz + ps.tL[1];
    const double lz = ps.RL[6] * bx + ps.RL[7] * by + ps.RL[8] * bz + ps.tL[2];
    const float wx = (float)(ps.R[0] * lx + ps.R[1] * ly + ps.R[2] * lz + ps.t[0]);
    const float wy = (float)(ps.R[3] * lx + ps.R[4] * ly + ps.R[5] * lz + ps.t[1]);
    const float wz = (float)(ps.R[6] * lx + ps.R[7] * ly + ps.R[8] * lz + ps.t[2]);
    world[i] = make_float4(wx, wy, wz, pb.w);
    float pabcd[4] = {0.f, 0.f, 0.f, 0.f};
    bool ok = false;
    if (FIT) {
      if (near_cnt[i] >= 5) {  // point_selected_surf, laserMapping.cpp:847,850
        float px[5], py[5], pz[5];
#pragma unroll
        for (int j = 0; j < 5; j++) { const float4 q = near[(size_t)i * 5 + j]; px[j] = q.x; py[j] = q.y; pz[j] = q.z; }
        ok = esti_plane_dev(px, py, pz, 0.1f, pabcd);
      }
      pabcd_io[i] = make_float4(pabcd[0], pabcd[1], pabcd[2], pabcd[3]);
      plane_ok[i] = ok ? 1 : 0;
    } else if (selected[i] && plane_ok[i]) {
      const float4 pl = pabcd_io[i];
      pabcd[0] = pl.x; pabcd[1] = pl.y; pabcd[2] = pl.z; pabcd[3] = pl.w;
      ok = true;
    }
    bool keep = false;
    if (ok) {
      const float pd2 = pabcd[0] * wx + pabcd[1] * wy + pabcd[2] * wz + pabcd[3];
      const double s = 1 - 0.9 * fabs((double)pd2) / sqrt(sqrt(bx * bx + by * by + bz * bz));  // laserMapping.cpp:861
      if ((float)s > 0.9) {
        keep = true;
        plane[i] = make_float4(pabcd[0], pabcd[1], pabcd[2], pd2);
        const RowH r = make_row(ps, lx, ly, lz, pabcd, pd2);
        int q = 0;
#pragma unroll
        for (int a = 0; a < 6; a++) {
#pragma unroll
          for (int c = a; c < 6; c++) vals[q++] += r.row[a] * r.row[c];
        }
#pragma unroll
        for (int a = 0; a < 6; a++) vals[21 + a] += r.row[a] * r.h;
        vals[27] += (double)fabsf(pd2);  // res_last
        vals[28] += 1.0;
      }
    }
    selected[i] = keep ? 1 : 0;
  }
  block_partials<29>(vals, partials);
  grid_finalize<29>(partials, done, result, 0, 29, (double)n_true, kResSeq, seq, sc, 0);
}

// ---------------------------------------------------------------- K4+K5, reuse evaluation, ONE thread-block cluster
// Iterations that keep Nearest_Points (ekfom_data.converge == false, laserMapping.cpp:842) only re-evaluate the cached
// planes: ~12 k points x ~200 flops.  The grid-wide shape above spends most of its 15 us on launch + drain + the
// partials -> atomic ticket -> last-block fold chain.  Here the whole evaluation is ONE cluster of 8 CTAs x 1024 threads
// (8192 points per pass): warp shuffles -> per-warp accumulators in shared memory -> one partial vector per CTA written
// into CTA 0's shared memory over DSMEM -> cluster barrier -> CTA 0 folds the 8 vectors in rank order and publishes to
// the host.  No global partials, no atomics, no __threadfence; fixed order, so bit-reproducible.  Single-GPU handles only
// (the tile-sharded mode keeps the grid-wide kernel and its in-kernel cross-rank exchange).
#ifndef LSD_SIMT_EMU
}  // namespace lsd
#include <cooperative_groups.h>
namespace lsd {
namespace cg = cooperative_groups;
constexpr int kRcMaxCtas = 16, kRcMaxWarps = 32;   // cluster shape chosen at launch (lsd_lio::rc_ctas x rc_threads)
__global__ void __launch_bounds__(1024, 1)
lio_hmodel_reuse_cluster_kernel(const float4* __restrict__ body, const int* __restrict__ n_ptr, int cap, LioPose ps,
                                unsigned char* __restrict__ selected, const float4* __restrict__ pabcd_io,
                                const unsigned char* __restrict__ plane_ok, float4* __restrict__ plane, float4* __restrict__ world,
                                double* __restrict__ result, double seq) {
  pdl_enter();
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ double sm_w[kRcMaxWarps][30];    // per-warp accumulators
  __shared__ double sm_cta[kRcMaxCtas][32];   // CTA 0's copy collects one partial vector per CTA
  const int kRcCtas = (int)cluster.num_blocks(), kRcThreads = (int)blockDim.x, kRcWarps = kRcThreads >> 5;
  const int n_true = __ldcg(n_ptr);
  const int n = min(n_true, cap);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned rank = cluster.block_rank();
  if (lane < 30) sm_w[warp][lane] = 0.0;
  __syncwarp();
  const int stride = kRcCtas * kRcThreads;
  const int n_pass = (n + stride - 1) / stride;
#pragma unroll 1
  for (int pass = 0; pass < n_pass; pass++) {
    const int i = pass * stride + (int)rank * kRcThreads + (int)threadIdx.x;
    double row[6] = {0, 0, 0, 0, 0, 0}, h = 0.0, ares = 0.0, one = 0.0;
    if (i < n) {
      const float4 pb = __ldg(body + i);
      const double bx = pb.x, by = pb.y, bz = pb.z;
      const double lx = ps.RL[0] * bx + ps.RL[1] * by + ps.RL[2] * bz + ps.tL[0];
      const double ly = ps.RL[3] * bx + ps.RL[4] * by + ps.RL[5] * bz + ps.tL[1];
      const double lz = ps.RL[6] * bx + ps.RL[7] * by + ps.RL[8] * bz + ps.tL[2];
      const float wx = (float)(ps.R[0] * lx + ps.R[1] * ly + ps.R[2] * lz + ps.t[0]);
      const float wy = (float)(ps.R[3] * lx + ps.R[4] * ly + ps.R[5] * lz + ps.t[1]);
      const float wz = (float)(ps.R[6] * lx + ps.R[7] * ly + ps.R[8] * lz + ps.t[2]);
      world[i] = make_float4(wx, wy, wz, pb.w);
      bool keep = false;
      if (selected[i] && plane_ok[i]) {
        const float4 pl = pabcd_io[i];
        const float pabcd[4] = {pl.x, pl.y, pl.z, pl.w};
        const float pd2 = pabcd[0] * wx + pabcd[1] * wy + pabcd[2] * wz + pabcd[3];
        const double s = 1 - 0.9 * fabs((double)pd2) / sqrt(sqrt(bx * bx + by * by + bz * bz));  // laserMapping.cpp:861
        if ((float)s > 0.9) {
          keep = true;
          plane[i] = make_float4(pabcd[0], pabcd[1], pabcd[2], pd2);
          const RowH r = make_row(ps, lx, ly, lz, pabcd, pd2);
#pragma unroll
          for (int a = 0; a < 6; a++) row[a] = r.row[a];
          h = r.h; ares = (double)fabsf(pd2); one = 1.0;
        }
      }
      selected[i] = keep ? 1 : 0;
    }
    // 29 sums of this pass: products formed on the fly, warp tree, lane 0 accumulates (ascending passes)
    int q = 0;
#pragma unroll
    for (int a = 0; a < 6; a++) {
#pragma unroll
      for (int c = a; c < 6; c++) { const double v = warp_sum(row[a] * row[c]); if (lane == 0) sm_w[warp][q] += v; q++; }
    }
#pragma unroll
    for (int a = 0; a < 6; a++) { const double v = warp_sum(row[a] * h); if (lane == 0) sm_w[warp][21 + a] += v; }
    { const double v = warp_sum(ares); if (lane == 0) sm_w[warp][27] += v; }
    { const double v = warp_sum(one); if (lane == 0) sm_w[warp][28] += v; }
  }
  __syncthreads();
  if (threadIdx.x < 29) {
    double s = 0.0;
    for (int w = 0; w < kRcWarps; w++) s += sm_w[w][threadIdx.x];
    double* dst = cluster.map_shared_rank(&sm_cta[0][0], 0);     // CTA 0's shared memory, over DSMEM
    dst[rank * 32 + threadIdx.x] = s;
  }
  cluster.sync();
  if (rank == 0) {
    if (threadIdx.x < 29) {
      double t = 0.0;
      for (int r = 0; r < kRcCtas; r++) t += sm_cta[r][threadIdx.x];
      reinterpret_cast<volatile double*>(result)[threadIdx.x] = t;
      __threadfence_system();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      volatile double* res = result;
      res[29] = (double)n_true;
      __threadfence_system();
      res[kResSeq] = seq;  // published last
    }
  }
}
#endif

// ---------------------------------------------------------------- degeneracy sums (laserMapping.cpp:946-970)
// Only launched when the host cannot certify non-degeneracy from the eigenvalues (lio_linearize).
struct Eig3 { double V[9]; };  // columns = eigenvectors
__global__ void __launch_bounds__(kLioBlock) lio_degen_kernel(const int* __restrict__ n_ptr, int cap,
                                                              const unsigned char* __restrict__ selected,
                                                              const float4* __restrict__ plane, Eig3 e, double* __restrict__ partials,
                                                              unsigned* __restrict__ done, double* __restrict__ result, double seq,
                                                              ShardComm sc) {
  pdl_enter();
  const int n = min(__ldcg(n_ptr), cap);
  const double* V = e.V;
  double vals[6] = {0, 0, 0, 0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!selected[i]) continue;
    const float4 p = plane[i];
    const double r0 = p.x, r1 = p.y, r2 = p.z;
    const double nn = sqrt(r0 * r0 + r1 * r1 + r2 * r2);
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const float dotp = (float)fabs((r0 / nn) * V[k] + (r1 / nn) * V[3 + k] + (r2 / nn) * V[6 + k]);
      if (dotp > 0.1736) vals[k] += dotp;
      if (dotp > 0.7070) vals[3 + k] += dotp;
    }
  }
  block_partials<6>(vals, partials);
  grid_finalize<6>(partials, done, result, kResDegen, -1, 0.0, kResSeqDegen, seq, sc, 1);
}

// ---------------------------------------------------------------- map_incremental (laserMapping.cpp:523-576)
__device__ __forceinline__ float calc_dist3(float ax, float ay, float az, float bx, float by, float bz) {
  return (ax - bx) * (ax - bx) + (ay - by) * (ay - by) + (az - bz) * (az - bz);
}
__global__ void __launch_bounds__(256) lio_map_incremental_kernel(MapView mv, const float4* __restrict__ body,
                                                                  const int* __restrict__ n_ptr, int cap, LioPose ps,
                                                                  const float4* __restrict__ near, const int* __restrict__ near_cnt,
                                                                  int ekf_inited, double fsize, int id0, int id_t2, int use_near,
                                                                  float4* __restrict__ world, unsigned char* __restrict__ flags,
                                                                  unsigned* __restrict__ n_added, ShardComm sc, double seq,
                                                                  unsigned* __restrict__ done) {
  pdl_enter();
  const int n = min(__ldcg(n_ptr), cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float4 pb = __ldg(body + i);
    const double bx = pb.x, by = pb.y, bz = pb.z;
    const double lx = ps.RL[0] * bx + ps.RL[1] * by + ps.RL[2] * bz + ps.tL[0];
    const double ly = ps.RL[3] * bx + ps.RL[4] * by + ps.RL[5] * bz + ps.tL[1];
    const double lz = ps.RL[6] * bx + ps.RL[7] * by + ps.RL[8] * bz + ps.tL[2];
    const float wx = (float)(ps.R[0] * lx + ps.R[1] * ly + ps.R[2] * lz + ps.t[0]);
    const float wy = (float)(ps.R[3] * lx + ps.R[4] * ly + ps.R[5] * lz + ps.t[1]);
    const float wz = (float)(ps.R[6] * lx + ps.R[7] * ly + ps.R[8] * lz + ps.t[2]);
    world[i] = make_float4(wx, wy, wz, pb.w);
    bool mine = true;
    if (sc.world > 1) { const int3 hc = pos2grid(wx, wy, wz, mv.inv_res); mine = shard_owns(mv, hc.x, hc.y); }
    if (mine) {
      int f = 1;  // PointToAdd
      const int cnt = use_near ? near_cnt[i] : 0;
      if (cnt > 0 && ekf_inited) {
        const float mx = (float)(floor((double)wx / fsize) * fsize + 0.5 * fsize);
        const float my = (float)(floor((double)wy / fsize) * fsize + 0.5 * fsize);
        const float mz = (float)(floor((double)wz / fsize) * fsize + 0.5 * fsize);
        const float dist = calc_dist3(wx, wy, wz, mx, my, mz);
        const float4 n0 = near[(size_t)i * 5];
        if ((double)fabsf(n0.x - mx) > 0.5 * fsize && (double)fabsf(n0.y - my) > 0.5 * fsize && (double)fabsf(n0.z - mz) > 0.5 * fsize) {
          f = 2;  // PointNoNeedDownsample
        } else if (cnt >= 5) {
#pragma unroll
          for (int r = 0; r < 5; r++) {
            const float4 q = near[(size_t)i * 5 + r];
            if (calc_dist3(q.x, q.y, q.z, mx, my, mz) < dist) f = 0;
          }
        }
      }
      flags[i] = (unsigned char)f;
      if (f) {
        // id_t2 (reference-order mode): ids grow in the reference's insertion order — every PointToAdd of a scan before
        // every PointNoNeedDownsample (laserMapping.cpp:571-572) — because a voxel's points_ order is part of the
        // candidate sequence GetClosestPoint hands to nth_element
        map_insert_point(mv, wx, wy, wz, id0 + i + (f == 2 ? id_t2 : 0));
        atomicAdd(n_added, 1u);
      }
      // halo exchange, step 1: tell every other rank what was decided for this point
      for (int p = 0; p < sc.world; p++) if (p != sc.rank) sc.flagbox[p][i] = (unsigned char)f;
    }
  }
  if (sc.world > 1) {  // last block: all decisions of this rank are out -> publish the sequence number
    __shared__ bool is_last;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(done, 1u) == gridDim.x - 1;
    __syncthreads();
    if (is_last && threadIdx.x < sc.world) {
      volatile unsigned long long* d = reinterpret_cast<volatile unsigned long long*>(sc.flagbox[threadIdx.x] + cap) + sc.rank;
      *d = (unsigned long long)seq;
      __threadfence_system();
      if (threadIdx.x == 0) *done = 0u;
    }
  }
}

// halo exchange, step 2: insert the points other ranks decided to add that fall in this rank's halo
// (their world coordinates are known locally: every rank holds the whole downsampled scan).
__global__ void __launch_bounds__(256) lio_halo_insert_kernel(MapView mv, const int* __restrict__ n_ptr, int cap,
                                                              const float4* __restrict__ world, int id0, int id_t2, ShardComm sc, double seq,
                                                              unsigned* __restrict__ n_added) {
  pdl_enter();
  __shared__ int ready;
  if (threadIdx.x < sc.world && threadIdx.x != sc.rank) {
    volatile unsigned long long* d = reinterpret_cast<volatile unsigned long long*>(sc.flagbox[sc.rank] + cap) + threadIdx.x;
    while (*d != (unsigned long long)seq) {}
  }
  if (threadIdx.x == 0) ready = 1;
  __syncthreads();
  __threadfence_system();
  const int n = min(__ldcg(n_ptr), cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !ready) return;
  const float4 w = world[i];
  const int3 hc = pos2grid(w.x, w.y, w.z, mv.inv_res);
  if (shard_owns(mv, hc.x, hc.y) || !shard_relevant(mv, hc.x, hc.y)) return;
  const unsigned char f = *(volatile unsigned char*)(sc.flagbox[sc.rank] + i);
  if (f == 1 || f == 2) {
    map_insert_point(mv, w.x, w.y, w.z, id0 + i + (f == 2 ? id_t2 : 0));
    atomicAdd(n_added, 1u);
  }
}

__global__ void lio_fill_u8_kernel(unsigned char* p, int n, unsigned char v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void lio_set_int_kernel(int* p, int v) { *p = v; }
// a default-constructed Nearest_Points: empty rows (ids -1)
__global__ void lio_clear_rows_kernel(float4* near, int* near_cnt, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  near_cnt[i] = 0;
#pragma unroll
  for (int r = 0; r < 5; r++) near[(size_t)i * 5 + r] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
}

// ---------------------------------------------------------------- host side
static void pose_from_state(const double* x, LioPose* ps) {
  eskf::q2R(x + eskf::S_ROT, ps->R);
  eskf::q2R(x + eskf::S_OFFR, ps->RL);
  for (int i = 0; i < 3; i++) { ps->t[i] = x[eskf::S_POS + i]; ps->tL[i] = x[eskf::S_OFFT + i]; }
}

struct ProfScope {  // CUDA-event timing of one launch group on the LIO stream (profile mode only)
  lsd_lio* l; int kind; bool on;
  ProfScope(lsd_lio* l_, int kind_) : l(l_), kind(kind_), on(l_->profile != 0) { if (on) cudaEventRecord(l->pev[0], l->stream); }
  void stop() {
    if (!on) return;
    cudaEventRecord(l->pev[1], l->stream);
    cudaEventSynchronize(l->pev[1]);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, l->pev[0], l->pev[1]);
    l->prof_ms[kind] += ms; l->prof_cnt[kind]++;
    on = false;
  }
};

// Spin on the sequence number a kernel publishes into mapped host memory at `slot`.  The load is an acquire: the sums the
// kernel stored before the sequence number must not be read ahead of it (aarch64 hosts reorder loads).  Bounded by a
// wall-clock limit so that a hung kernel (e.g. a peer that never answers the in-kernel all-reduce) becomes an error.
// Used by the LIO front end, the matcher (reg.cu) and the loop detector (loop.cu).
static lsd_status_t wait_seq(const double* slot, cudaStream_t stream, double seq, double timeout_s) {
  const unsigned long long* h = reinterpret_cast<const unsigned long long*>(slot);
  unsigned long long want;
  memcpy(&want, &seq, 8);
  const auto t0 = std::chrono::steady_clock::now();
  for (unsigned long long spins = 0;; spins++) {
    if (__atomic_load_n(h, __ATOMIC_ACQUIRE) == want) return LSD_OK;
    if ((spins & 0xfff) == 0xfff) {
      cudaError_t e = cudaStreamQuery(stream);
      if (e != cudaSuccess && e != cudaErrorNotReady) return cuda_fail(e, "kernel while waiting for the reduction", __FILE__, __LINE__);
      if (e == cudaSuccess) {  // stream drained: the result must be there
        if (__atomic_load_n(h, __ATOMIC_ACQUIRE) == want) return LSD_OK;
        set_error("reduction result never published");
        return LSD_ERR_CUDA;
      }
      if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > timeout_s) {
        set_error("timed out after %.0f s waiting for a reduction result (kernel hung?)", timeout_s);
        return LSD_ERR_CUDA;
      }
    }
  }
}

static int grid_for(int n) { return std::max(1, std::min((n + kLioBlock - 1) / kLioBlock, kLioMaxGrid)); }

static lsd_status_t issue_deferred_prefetch(lsd_lio* l);

// One h_share_model_geometric evaluation on the loaded scan.  Fills HTH6/HTh6 (after the
// degeneracy projection when it triggers).  One host synchronisation per evaluation.
lsd_status_t lio_linearize(lsd_lio* l, const double* x, bool search, double* HTH6, double* HTh6, double* res_sum,
                           int* n_eff, int* degenerate) {
  LioPose ps;
  pose_from_state(x, &ps);
  cudaStream_t st = l->stream;
  const int stencil = l->p.knn_mode_exact ? LSD_STENCIL_EXACT : l->p.ivox_nearby;
  const double seq = (double)(++l->seq);
  const int pdl = l->pdl && l->sc.world <= 1;   // programmatic dependent launch (lsd_lio_set_pdl); single-GPU chains only
  ProfScope prof(l, search ? 0 : 1);
  if (search) {
    const int keep_stale = (l->stale_rows && !l->p.knn_mode_exact && l->map->view.shard_world <= 1) ? 1 : 0;
    const int ref_order = (l->reference_order && !l->p.knn_mode_exact && l->d_ref_fallbacks) ? 1 : 0;
    int resize_parity = -1;
    if (l->rows_resize_pending) { resize_parity = l->rows_parity; l->rows_parity ^= 1; l->rows_resize_pending = false; }
    const int nb = std::max(1, std::min((l->n_bound + kHmWarps - 1) / kHmWarps, l->max_search_blocks));
    LSD_LAUNCH(pdl, lio_knn_kernel, nb, kHmWarps * 32, st, l->map->view, stencil, l->d_body, l->d_n, l->p.max_points, ps, l->d_near, l->d_near_cnt,
               keep_stale, l->d_rows, resize_parity, ref_order, l->d_ref_fallbacks);
    LSD_LAUNCH(pdl, lio_hmodel_kernel<true>, grid_for(l->n_bound), kLioBlock, st, l->d_body, l->d_n, l->p.max_points, ps, l->d_near, l->d_near_cnt,
               l->d_selected, l->d_pabcd, l->d_plane_ok, l->d_plane, l->d_world,
               l->d_partials, l->d_done, l->d_result, seq, l->sc);
    l->launches += 2;
  } else {
#ifndef LSD_SIMT_EMU
    if (l->sc.world <= 1 && l->reuse_cluster) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(l->rc_ctas); cfg.blockDim = dim3(l->rc_threads); cfg.dynamicSmemBytes = 0; cfg.stream = st;
      cudaLaunchAttribute at[2];
      int na = 0;
      at[na].id = cudaLaunchAttributeClusterDimension; at[na].val.clusterDim.x = l->rc_ctas; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1; na++;
      if (pdl) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; na++; }
      cfg.attrs = at; cfg.numAttrs = na;
      (void)cudaLaunchKernelEx(&cfg, lio_hmodel_reuse_cluster_kernel, (const float4*)l->d_body, (const int*)l->d_n, l->p.max_points, ps, l->d_selected,
                               (const float4*)l->d_pabcd, (const unsigned char*)l->d_plane_ok, l->d_plane, l->d_world, l->d_result, seq);
    } else
#endif
    LSD_LAUNCH(pdl, lio_hmodel_kernel<false>, grid_for(l->n_bound), kLioBlock, st, l->d_body, l->d_n, l->p.max_points, ps, l->d_near, l->d_near_cnt,
               l->d_selected, l->d_pabcd, l->d_plane_ok, l->d_plane, l->d_world,
               l->d_partials, l->d_done, l->d_result, seq, l->sc);
    l->launches++;
  }
  LSD_CUDA(cudaGetLastError());
  prof.stop();
  if (l->issue_in_linearize) { lsd_status_t d = issue_deferred_prefetch(l); if (d) return d; }   // hidden under this evaluation
  { lsd_status_t w = wait_seq(l->h_result + kResSeq, l->stream, seq, l->wait_timeout_s); if (w) return w; }
  const double* r = l->h_result;
  if (l->sc.world > 1) { l->xchg_cycles += r[kResWaitCycles]; l->xchg_count++; }
  int q = 0;
  for (int a = 0; a < 6; a++) for (int c = a; c < 6; c++) { HTH6[6 * a + c] = HTH6[6 * c + a] = r[q]; q++; }
  for (int a = 0; a < 6; a++) HTh6[a] = r[21 + a];
  *res_sum = r[27];
  *n_eff = (int)(r[28] + 0.5);
  l->n_down = (int)(r[29] + 0.5);
  if (l->n_down > l->p.max_points) { set_error("downsampled scan of %d points exceeds max_points %d", l->n_down, l->p.max_points); return LSD_ERR_CAPACITY; }
  l->n_bound = std::max(l->n_down, 1);  // later launches cover exactly the downsampled scan
  *degenerate = 0;
  if (*n_eff < 1) return LSD_NO_EFFECTIVE_POINTS;
  if (l->p.degenerate_detect_en) {
    // Degeneracy detection (laserMapping.cpp:934-980).  For an eigenvector v_k of the 3x3 normal
    // block, sum_j (n_j . v_k)^2 = lambda_k because the rows are unit normals, hence
    //   local_contri_k = sum_{|n.v| > 0.1736} |n.v| >= lambda_k - 0.1736^2 * n_eff.
    // When that bound already clears the 250 threshold for every k the scan is certified
    // non-degenerate without touching the points again; otherwise the exact sums are computed.
    double H3[9], V[9], w[3];
    for (int a = 0; a < 3; a++) for (int c = 0; c < 3; c++) H3[3 * a + c] = HTH6[6 * a + c];
    eig3_sym(H3, V, w);
    const double wmin = std::min(w[0], std::min(w[1], w[2]));
    if (wmin - 0.0302 * (double)*n_eff < 260.0) {
      Eig3 e;
      memcpy(e.V, V, sizeof(V));
      LSD_LAUNCH(pdl, lio_degen_kernel, grid_for(l->n_bound), kLioBlock, st, l->d_n, l->p.max_points, l->d_selected, l->d_plane, e, l->d_partials,
                 l->d_done, l->d_result, seq, l->sc);
      LSD_CUDA(cudaGetLastError());
      l->launches++;
      { lsd_status_t w = wait_seq(l->h_result + kResSeqDegen, l->stream, seq, l->wait_timeout_s); if (w) return w; }
      const double* dg = l->h_result + kResDegen;
      int mask[3] = {1, 1, 1};
      bool deg = false;
      for (int k = 0; k < 3; k++)
        if ((float)dg[k] < 250.0f && (float)dg[3 + k] < 50.0f) { mask[k] = 0; deg = true; }
      if (deg) {
        // rows n -> Pm n with Pm = V diag(mask) V^T  (mat_p, laserMapping.cpp:975-978):
        // HTH <- B HTH B^T, HTh <- B HTh with B = blockdiag(Pm, I3)
        double Pm[9] = {0};
        for (int a = 0; a < 3; a++) for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) if (mask[k]) Pm[3 * a + c] += V[3 * a + k] * V[3 * c + k];
        double B[36] = {0}, T[36];
        for (int a = 0; a < 3; a++) for (int c = 0; c < 3; c++) B[6 * a + c] = Pm[3 * a + c];
        for (int a = 3; a < 6; a++) B[6 * a + a] = 1.0;
        for (int a = 0; a < 6; a++) for (int c = 0; c < 6; c++) { double sum = 0; for (int k = 0; k < 6; k++) sum += B[6 * a + k] * HTH6[6 * k + c]; T[6 * a + c] = sum; }
        for (int a = 0; a < 6; a++) for (int c = 0; c < 6; c++) { double sum = 0; for (int k = 0; k < 6; k++) sum += T[6 * a + k] * B[6 * c + k]; HTH6[6 * a + c] = sum; }
        double h2[6];
        for (int a = 0; a < 6; a++) { double sum = 0; for (int k = 0; k < 6; k++) sum += B[6 * a + k] * HTh6[k]; h2[a] = sum; }
        memcpy(HTh6, h2, sizeof(h2));
        memcpy(l->last_Pm, Pm, sizeof(Pm));
        *degenerate = 1;
      }
    }
  }
  return LSD_OK;
}

// Rows of h_x for the rare n_eff < 23 branch of the filter (esekfom.hpp:1727): rebuilt on the host
// from the per-point taps.
static lsd_status_t fetch_rows(lsd_lio* l, const double* x, bool degenerate, std::vector<double>* h_x, std::vector<double>* h) {
  const int n = l->n_down;
  std::vector<float4> body(n), plane(n);
  std::vector<unsigned char> sel(n);
  LSD_CUDA(cudaMemcpyAsync(body.data(), l->d_body, (size_t)n * 16, cudaMemcpyDeviceToHost, l->stream));
  LSD_CUDA(cudaMemcpyAsync(plane.data(), l->d_plane, (size_t)n * 16, cudaMemcpyDeviceToHost, l->stream));
  LSD_CUDA(cudaMemcpyAsync(sel.data(), l->d_selected, (size_t)n, cudaMemcpyDeviceToHost, l->stream));
  LSD_CUDA(cudaStreamSynchronize(l->stream));
  LioPose ps;
  pose_from_state(x, &ps);
  h_x->clear(); h->clear();
  for (int i = 0; i < n; i++) {
    if (!sel[i]) continue;
    const double bx = body[i].x, by = body[i].y, bz = body[i].z;
    const double lx = ps.RL[0] * bx + ps.RL[1] * by + ps.RL[2] * bz + ps.tL[0];
    const double ly = ps.RL[3] * bx + ps.RL[4] * by + ps.RL[5] * bz + ps.tL[1];
    const double lz = ps.RL[6] * bx + ps.RL[7] * by + ps.RL[8] * bz + ps.tL[2];
    double nv[3] = {plane[i].x, plane[i].y, plane[i].z};
    const double cx = ps.R[0] * nv[0] + ps.R[3] * nv[1] + ps.R[6] * nv[2];
    const double cy = ps.R[1] * nv[0] + ps.R[4] * nv[1] + ps.R[7] * nv[2];
    const double cz = ps.R[2] * nv[0] + ps.R[5] * nv[1] + ps.R[8] * nv[2];
    if (degenerate) { double o[3]; eskf::mv3(l->last_Pm, nv, o); nv[0] = o[0]; nv[1] = o[1]; nv[2] = o[2]; }
    double row[15] = {nv[0], nv[1], nv[2], ly * cz - lz * cy, lz * cx - lx * cz, lx * cy - ly * cx, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    h_x->insert(h_x->end(), row, row + 15);
    h->push_back(-(double)plane[i].w);
  }
  return LSD_OK;
}

lsd_status_t lio_update(lsd_lio* l, double* x, double* P, lsd_lio_info_t* info) {
  lsd_status_t err = LSD_OK;
  int last_neff = 0, last_deg = 0;
  double last_res = 0.0;
  auto hm = [&](const double* xs, bool converge, eskf::HModel* out) {
    double HTH6[36], HTh6[6], rs;
    int ne, dg;
    lsd_status_t s = lio_linearize(l, xs, converge, HTH6, HTh6, &rs, &ne, &dg);
    if (s < 0) { err = s; out->valid = false; return; }
    if (l->n_down < 5) { out->valid = false; return; }  // laserMapping.cpp:1252-1256: scan skipped, state untouched
    last_neff = ne; last_deg = dg; last_res = ne > 0 ? rs / ne : 0.0;
    out->valid = ne >= 1;
    out->n = ne;
    if (!out->valid) return;
    memset(out->HTH, 0, sizeof(out->HTH)); memset(out->HTh, 0, sizeof(out->HTh));
    for (int a = 0; a < 6; a++) { for (int c = 0; c < 6; c++) out->HTH[15 * a + c] = HTH6[6 * a + c]; out->HTh[a] = HTh6[a]; }
    if (ne < eskf::N) { lsd_status_t f = fetch_rows(l, xs, dg != 0, &out->h_x, &out->h); if (f < 0) { err = f; out->valid = false; } }
  };
  eskf::UpdateResult r = eskf::update_iterated(x, P, hm, l->p.laser_point_cov, l->p.max_iterations, l->p.converge_eps, l->p.eskf_literal != 0);
  if (info) {
    info->iterations = r.evaluations; info->n_eff = last_neff; info->degenerate = last_deg; info->res_mean = last_res;
    info->converged = r.returned_converged ? 1 : 0; info->n_down = l->n_down;
  }
  if (err < 0) return err;
  return last_neff >= 1 ? LSD_OK : LSD_NO_EFFECTIVE_POINTS;
}

// Collect what an asynchronous lio_scan left pending (device time and insert count of that scan).
static lsd_status_t lio_drain(lsd_lio* l) {
  if (!l->pending) return LSD_OK;
  LSD_CUDA(cudaEventSynchronize(l->ev1));
  float ms = 0.f;
  LSD_CUDA(cudaEventElapsedTime(&ms, l->ev0, l->ev1));
  l->last_gpu_ms = ms;
  l->last_added = (int)*l->h_added;
  l->pending = false;
  return LSD_OK;
}

// map_incremental on the stream; with wait == false the insert count is copied to pinned memory
// asynchronously and picked up by lio_drain().
lsd_status_t lio_map_incremental(lsd_lio* l, const double* x, int use_near, int* n_added, bool wait) {
  LioPose ps;
  pose_from_state(x, &ps);
  cudaStream_t st = l->stream;
  LSD_CUDA(cudaMemsetAsync(l->d_added, 0, sizeof(unsigned), st));
  ProfScope prof(l, 3);
  const int nb = std::max(1, (l->n_bound + 255) / 256);
  const double mseq = (double)(++l->mi_seq);
  const int pdl = 0;   // its stream predecessor is the memset above, not a kernel: nothing to hide, so keep the plain launch
  const int id_t2 = (l->reference_order && use_near) ? l->n_bound : 0;   // reference-order mode: a registered scan takes 2 x n ids (type 1 block, type 2 block)
  LSD_LAUNCH(pdl, lio_map_incremental_kernel, nb, 256, st, l->map->view, l->d_body, l->d_n, l->p.max_points, ps, l->d_near, l->d_near_cnt, l->ekf_inited,
             (double)l->p.filter_size_map, l->next_id, id_t2, use_near, l->d_world, l->d_flags, l->d_added,
             l->sc, mseq, l->d_done);
  LSD_CUDA(cudaGetLastError());
  l->launches++;
  if (l->sc.world > 1) {
    lio_halo_insert_kernel<<<nb, 256, 0, st>>>(l->map->view, l->d_n, l->p.max_points, l->d_world, l->next_id, id_t2, l->sc, mseq, l->d_added);
    LSD_CUDA(cudaGetLastError());
    l->launches++;
  }
  prof.stop();
  LSD_CUDA(cudaMemcpyAsync(l->h_added, l->d_added, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaMemcpyAsync(l->h_added + 2, &l->map->view.counters[2], sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));   // points the map refused so far
  if (l->map->lru && l->sc.world <= 1) {
    // iVox's LRU (lsd_map_enable_lru): replay this scan's AddPoints calls on the host mirror in the reference's order —
    // PointToAdd first, then PointNoNeedDownsample (laserMapping.cpp:571-572), both at this scan's travel distance —
    // and apply the evictions before the next search can see the map.
    const int n = std::max(l->n_down, 0);
    std::vector<float4> w((size_t)n);
    std::vector<unsigned char> f((size_t)n);
    if (n) {
      LSD_CUDA(cudaMemcpyAsync(w.data(), l->d_world, (size_t)n * 16, cudaMemcpyDeviceToHost, st));
      LSD_CUDA(cudaMemcpyAsync(f.data(), l->d_flags, (size_t)n, cudaMemcpyDeviceToHost, st));
    }
    LSD_CUDA(cudaStreamSynchronize(st));
    std::vector<float4> pts; std::vector<int> ids;
    for (int pass = 1; pass <= 2; pass++)
      for (int i = 0; i < n; i++) if (f[i] == pass) { pts.push_back(w[i]); ids.push_back(l->next_id + i + (pass == 2 ? id_t2 : 0)); }
    l->map->lru->distance = l->travel;
    lsd_status_t e = map_lru_touch(l->map, pts.data(), ids.data(), (int)pts.size(), 0, st);
    if (e) return e;
    wait = true;
  }
  // ids are 31-bit labels (-1 = no point): wrap instead of overflowing.  After a wrap — 2^31 / (2 n) scans, ~2.5 h at 10 Hz and
  // 12 k points per scan — a voxel that still holds points from before it orders them after the new ones (reference-order
  // mode only; with iVox's LRU on, nothing that old survives 100 m of travel).
  l->next_id = (int)(((long long)l->next_id + l->n_bound + id_t2) & 0x7fffffffll);
  if (wait) {
    LSD_CUDA(cudaStreamSynchronize(st));
    if (n_added) *n_added = (int)*l->h_added;
  } else if (n_added) {
    *n_added = -1;
  }
  return LSD_OK;
}

lsd_status_t lio_load(lsd_lio* l, const float4* d_scan, int n, int downsample) {
  cudaStream_t st = l->stream;
  if (n < 0 || n > l->p.max_scan_points) { set_error("scan of %d points exceeds max_scan_points %d", n, l->p.max_scan_points); return LSD_ERR_CAPACITY; }
  lsd_lio::Stage* pre = l->pre;
  l->pre = nullptr;
  if (downsample && pre && pre->down) {
    // downsampled on the copy stream while the previous scan iterated (issue_side_vg); the caller made the stream wait
    // for pre->ev.  The buffers change hands: this scan's feats_down_body / size are the stage's, and the stage gets the
    // previous scan's (idle once everything queued on the stream so far has run, which the next side voxel grid waits for).
    std::swap(l->d_body, pre->body);
    std::swap(l->d_n, pre->dn);
    pre->down = false;
    l->side_vg_adopted++;
    l->n_bound = std::min(n, l->p.max_points);
    l->n_down = -1;
  } else if (downsample) {
    if (l->side_vg_inflight) {   // the voxel grid's scratch is shared with the copy stream's instance
      LSD_CUDA(cudaStreamWaitEvent(st, l->ev_side_vg, 0));
      l->side_vg_inflight = false;
    }
    ProfScope prof(l, 2);
    l->vg->pdl = (l->pdl && l->sc.world <= 1) ? 1 : 0;
    lsd_status_t s = vg_run(l->vg, d_scan, n, l->p.filter_size_surf, l->d_body, l->d_n, st);
    if (s) return s;
    prof.stop();
    l->launches += l->vg->input_order_sums ? 8 : 5;
    l->n_bound = std::min(n, l->p.max_points);
    l->n_down = -1;  // learned with the first reduction (or lsd_lio_load_scan's explicit read)
  } else {
    if (n > l->p.max_points) { set_error("scan of %d points exceeds max_points %d", n, l->p.max_points); return LSD_ERR_CAPACITY; }
    LSD_CUDA(cudaMemcpyAsync(l->d_body, d_scan, (size_t)n * 16, cudaMemcpyDeviceToDevice, st));
    lio_set_int_kernel<<<1, 1, 0, st>>>(l->d_n, n);
    l->launches++;
    l->n_bound = std::max(n, 1);
    l->n_down = n;
  }
  l->rows_resize_pending = l->stale_rows && l->map->view.shard_world <= 1;   // done by this scan's first search (lio_knn_kernel)
  return LSD_OK;
}

static lsd_status_t read_n_down(lsd_lio* l) {
  int h = 0;
  LSD_CUDA(cudaMemcpyAsync(&h, l->d_n, sizeof(int), cudaMemcpyDeviceToHost, l->stream));
  LSD_CUDA(cudaStreamSynchronize(l->stream));
  if (h > l->p.max_points) { set_error("downsampled scan of %d points exceeds max_points %d", h, l->p.max_points); return LSD_ERR_CAPACITY; }
  l->n_down = h;
  l->n_bound = std::max(h, 1);
  return LSD_OK;
}

// A prefetch request recorded by lsd_lio_prefetch is turned into the actual copy here, right after this scan's
// voxel-grid kernels were launched: the driver calls cost host time (~5 us) that is now hidden under GPU work
// instead of delaying the scan's first launch.  Target: the staging slot this scan does not read.
// Pipelined voxel grid (lsd_lio_set_pipeline): downsample the staged scan on the copy stream, behind its H2D copy, into the
// stage's own feats_down_body / size.  The voxel grid's scratch is shared with the main stream's instance, hence the event
// hand-shake: this one starts after everything queued on the main stream so far (the running scan's own voxel grid, the
// previous scan's map insert — the last reader of the buffer the stage now owns), and a later voxel grid on the main
// stream waits for ev_side_vg.  sg->ev is re-recorded behind the voxel grid, so the scan that adopts the stage waits once.
static lsd_status_t issue_side_vg(lsd_lio* l, lsd_lio::Stage* sg, const float4* src) {
  if (!l->main_ev_fresh) LSD_CUDA(cudaEventRecord(l->ev_main_vg, l->stream));   // else: recorded right behind this scan's load step
  l->main_ev_fresh = false;
  LSD_CUDA(cudaStreamWaitEvent(l->copy_stream, l->ev_main_vg, 0));
  l->vg->pdl = (l->pdl && l->sc.world <= 1) ? 1 : 0;
  lsd_status_t s = vg_run(l->vg, src, sg->n, l->p.filter_size_surf, sg->body, sg->dn, l->copy_stream);
  if (s) return s;
  l->launches += l->vg->input_order_sums ? 8 : 5;
  LSD_CUDA(cudaEventRecord(sg->ev, l->copy_stream));
  LSD_CUDA(cudaEventRecord(l->ev_side_vg, l->copy_stream));
  l->side_vg_inflight = true;
  l->side_vg_issued++;
  sg->down = true;
  return LSD_OK;
}

// A prefetch request recorded by lsd_lio_prefetch(_dev) is turned into the actual copy (and, pipelined, the voxel grid)
// here, once this scan's first kernels are in flight: the driver calls cost host time (~5 us, ~20 us with the voxel grid)
// that is hidden under GPU work instead of delaying the scan's first launch.  Target: the staging slot this scan does not read.
static lsd_status_t issue_deferred_prefetch(lsd_lio* l) {
  l->issue_in_linearize = false;
  if (!l->defer_pending) return LSD_OK;
  l->defer_pending = false;
  lsd_lio::Stage* sg = nullptr;
  for (int i = 0; i < 2; i++) if (i != l->busy_slot && !l->stage[i].valid) sg = &l->stage[i];
  if (!sg) return LSD_OK;  // both slots taken: the request is dropped, the later lsd_lio_scan uploads inline
  sg->down = false;
  sg->is_dev = l->defer_is_dev;
  sg->host = l->defer_host; sg->n = l->defer_n;
  const float4* src = reinterpret_cast<const float4*>(l->defer_host);
  if (!l->defer_is_dev) {
    LSD_CUDA(cudaMemcpyAsync(sg->buf, l->defer_host, (size_t)l->defer_n * 16, cudaMemcpyHostToDevice, l->copy_stream));
    LSD_CUDA(cudaEventRecord(sg->ev, l->copy_stream));
    src = sg->buf;
  }
  sg->valid = true; sg->age = ++l->stage_clock;
  // (tile-sharded handles included: the side voxel grid waits on nothing a peer produces, so it cannot hold up the
  // in-kernel exchange of the search kernels it overlaps with)
  if (l->pipeline_vg) return issue_side_vg(l, sg, src);
  return LSD_OK;
}

lsd_status_t lio_scan(lsd_lio* l, const float4* d_scan, int n, double* x, double* P, lsd_lio_info_t* info) {
  cudaStream_t st = l->stream;
  const long long launches0 = l->launches;
  const bool async = l->p.async_map_insert != 0;
  l->main_ev_fresh = false;   // (a scan that returned early on an error may have left it set)
  { lsd_status_t d = lio_drain(l); if (d) return d; }
  LSD_CUDA(cudaEventRecord(l->ev0, st));
  const bool adopted = l->pre && l->pre->down;
  lsd_status_t s = lio_load(l, d_scan, n, 1);
  if (s) return s;
  if (l->pipeline_vg && l->defer_pending) {
    // everything the next scan's voxel grid must wait for is queued by now (this scan's own voxel grid if it ran one, the
    // previous scan's map insert): mark the spot, so that it may overlap this scan's first evaluation too
    LSD_CUDA(cudaEventRecord(l->ev_main_vg, st));
    l->main_ev_fresh = true;
  }
  if (adopted) {
    l->issue_in_linearize = true;   // no voxel grid in flight to hide the driver calls behind: wait for the first search
  } else {
    s = issue_deferred_prefetch(l);
    if (s) return s;
  }
  lsd_lio_info_t inf;
  memset(&inf, 0, sizeof(inf));
  lsd_status_t ret = LSD_OK;
  uint64_t cells = l->map_cells_known;
  if (cells == 0) { s = lsd_map_stats(l->map, &cells, nullptr, nullptr); if (s) return s; l->map_cells_known = cells; }
  if (cells == 0) {  // first scan seeds the map (laserMapping.cpp:1227-1239)
    s = read_n_down(l);
    if (s) return s;
    inf.n_down = l->n_down;
    if (l->n_down > 5) { s = lio_map_incremental(l, x, 0, &inf.n_added, true); if (s) return s; l->map_cells_known = 1; }
    ret = LSD_MAP_SEEDED;
  } else {
    s = lio_update(l, x, P, &inf);
    if (s < 0) return s;
    if (l->n_down < 5) ret = LSD_SCAN_TOO_SMALL;  // laserMapping.cpp:1252-1256 (state untouched: n_eff == 0)
    else {
      ret = s;
      {  // travel_distance += |pos_lid - last_pos_lid| (laserMapping.cpp:1289-1291): what IVox::AddPoints ages voxels by
        double R[9], pl[3];
        eskf::q2R(x + eskf::S_ROT, R);
        for (int a = 0; a < 3; a++)
          pl[a] = x[eskf::S_POS + a] + R[3 * a] * x[eskf::S_OFFT] + R[3 * a + 1] * x[eskf::S_OFFT + 1] + R[3 * a + 2] * x[eskf::S_OFFT + 2];
        const double dx = pl[0] - l->last_pos_lid[0], dy = pl[1] - l->last_pos_lid[1], dz = pl[2] - l->last_pos_lid[2];
        l->travel += sqrt(dx * dx + dy * dy + dz * dz);
        for (int a = 0; a < 3; a++) l->last_pos_lid[a] = pl[a];
      }
      lsd_status_t m = lio_map_incremental(l, x, 1, &inf.n_added, !async);
      if (m) return m;
    }
  }
  if (l->issue_in_linearize) { s = issue_deferred_prefetch(l); if (s) return s; }   // no evaluation ran (seeding scan)
  l->main_ev_fresh = false;
  LSD_CUDA(cudaEventRecord(l->ev1, st));
  if (async && inf.n_added == -1) {
    // the pose is final; the map insert finishes in the background.  gpu_ms / n_added reported now
    // are those of the PREVIOUS scan (collected by lio_drain), see lsd_lio_params::async_map_insert.
    l->pending = true;
    inf.gpu_ms = l->last_gpu_ms;
    inf.n_added = l->last_added;
  } else {
    LSD_CUDA(cudaEventSynchronize(l->ev1));
    float ms = 0.f;
    LSD_CUDA(cudaEventElapsedTime(&ms, l->ev0, l->ev1));
    inf.gpu_ms = ms;
    l->last_gpu_ms = ms;
    l->last_added = inf.n_added;
  }
  inf.kernel_launches = (int)(l->launches - launches0);
  if (info) *info = inf;
  {  // a map that refuses points stops growing and odometry degrades silently: say so (one scan late with the async insert)
    const unsigned long long dropped = *reinterpret_cast<volatile unsigned long long*>(l->h_added + 2);
    if (dropped > l->map->dropped_seen) {
      l->map->dropped_seen = dropped;
      set_error("the map refused %llu points so far (hash table full along a probe chain, a voxel beyond 127 overflow lines, or coordinates beyond +-2^18 voxels): raise map_log2_lines or enable the LRU", dropped);
      if (ret == LSD_OK) ret = LSD_MAP_SATURATED;
    }
  }
  return ret;
}

}  // namespace lsd

using namespace lsd;

// a staging slot that holds no pending prefetch (else the older pending one, which is then dropped)
static lsd_lio::Stage* free_stage(lsd_lio* l) {
  for (int i = 0; i < 2; i++) if (!l->stage[i].valid) return &l->stage[i];
  lsd_lio::Stage* s = l->stage[0].age <= l->stage[1].age ? &l->stage[0] : &l->stage[1];
  // the dropped request's H2D copy (and side voxel grid) may still be running on the copy stream and reading s->buf:
  // whatever the caller queues on the main stream next has to wait for it
  cudaStreamWaitEvent(l->stream, s->ev, 0);
  s->valid = false; s->down = false;
  return s;
}

extern "C" {

void lsd_lio_default_params(lsd_lio_params_t* p) {
  if (!p) return;
  p->max_points = 100000;        // laserMapping.cpp:86,103
  p->max_scan_points = 400000;
  p->filter_size_surf = 0.5f;    // laserMapping.cpp:1027
  p->filter_size_map = 0.5f;     // laserMapping.cpp:1028
  p->ivox_resolution = 0.5f;     // laserMapping.cpp:1061
  p->ivox_nearby = LSD_STENCIL_NEARBY18;
  p->map_log2_lines = 22;
  p->max_iterations = 4;         // laserMapping.cpp:1026
  p->laser_point_cov = 0.001;    // laserMapping.cpp:71
  p->converge_eps = 0.001;       // laserMapping.cpp:1114-1116
  p->degenerate_detect_en = 1;   // laserMapping.cpp:83
  p->knn_mode_exact = 0;
  p->eskf_literal = 0;
  p->async_map_insert = 0;
}

lsd_status_t lsd_lio_create(lsd_lio_t** out, const lsd_lio_params_t* p) {
  if (!out || !p || p->max_points <= 0 || p->max_scan_points < p->max_points) { set_error("lsd_lio_create: bad params"); return LSD_ERR_INVALID; }
  lsd_status_t s = ensure_device();
  if (s) return s;
  lsd_lio* l = new lsd_lio();
  l->p = *p;
  memset(&l->sc, 0, sizeof(l->sc));
  l->sc.world = 1;
  cudaGetDevice(&l->device);
  s = lsd_map_create(&l->map, p->ivox_resolution, p->map_log2_lines);
  if (s) { delete l; return s; }
  s = lsd_voxelgrid_create(&l->vg, p->max_scan_points, 28);
  if (s) { lsd_map_destroy(l->map); delete l; return s; }
  const size_t mp = (size_t)p->max_points;
  const size_t max_blocks = (size_t)grid_for(p->max_points) + 1;
  l->max_search_blocks = lsd::kNumSms * 6;
  cudaError_t e = cudaStreamCreateWithFlags(&l->stream, cudaStreamNonBlocking);
  auto A = [&](void** ptr, size_t b) { if (e == cudaSuccess) e = cudaMalloc(ptr, b); if (e == cudaSuccess) e = cudaMemset(*ptr, 0, b); };
  for (int i = 0; i < 2; i++) {
    A((void**)&l->stage[i].buf, (size_t)p->max_scan_points * 16);
    A((void**)&l->stage[i].body, (size_t)p->max_scan_points * 16);   // pipelined voxel grid: the stage's feats_down_body / size
    A((void**)&l->stage[i].dn, 64);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&l->stage[i].ev, cudaEventDisableTiming);
  }
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&l->copy_stream, cudaStreamNonBlocking);
  A((void**)&l->d_body, (size_t)p->max_scan_points * 16);  // voxel-grid output may equal the input size
  A((void**)&l->d_n, 64);
  A((void**)&l->d_rows, 64);
  A((void**)&l->d_near, mp * 5 * 16);
  A((void**)&l->d_near_cnt, mp * 4);
  A((void**)&l->d_selected, mp);
  A((void**)&l->d_flags, mp);
  A((void**)&l->d_plane, mp * 16);
  A((void**)&l->d_pabcd, mp * 16);
  A((void**)&l->d_plane_ok, mp);
  A((void**)&l->d_world, mp * 16);
  A((void**)&l->d_partials, max_blocks * kNV * 8);
  A((void**)&l->d_done, 64);
  A((void**)&l->d_added, 64);
  if (e == cudaSuccess) e = cudaHostAlloc((void**)&l->h_result, kResDoubles * 8, cudaHostAllocMapped);
  if (e == cudaSuccess) { memset(l->h_result, 0, kResDoubles * 8); e = cudaHostGetDevicePointer((void**)&l->d_result, l->h_result, 0); }
  if (e == cudaSuccess) e = cudaMallocHost((void**)&l->h_added, 64);
  if (e == cudaSuccess) { memset(l->h_added, 0, 64); e = cudaEventCreate(&l->ev0); }
  if (e == cudaSuccess) e = cudaEventCreate(&l->ev1);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&l->ev_main_vg, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&l->ev_side_vg, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreate(&l->pev[0]);
  if (e == cudaSuccess) e = cudaEventCreate(&l->pev[1]);
  if (e == cudaSuccess) {  // memset(point_selected_surf, true), laserMapping.cpp:1089
    lio_fill_u8_kernel<<<(int)((mp + 255) / 256), 256, 0, l->stream>>>(l->d_selected, (int)mp, 1);
    lio_clear_rows_kernel<<<(int)((mp + 255) / 256), 256, 0, l->stream>>>(l->d_near, l->d_near_cnt, (int)mp);
    e = cudaStreamSynchronize(l->stream);
  }
  if (e != cudaSuccess) { lsd_status_t r = cuda_fail(e, "lsd_lio_create", __FILE__, __LINE__); lsd_lio_destroy(l); return r; }
  // the map and the voxel grid run on the LIO stream
  cudaStreamDestroy(l->map->stream); l->map->stream = l->stream;
  cudaStreamDestroy(l->vg->stream); l->vg->stream = l->stream;
  // The voxel grid of an announced scan is pipelined under the running one by default (bit-identical results,
  // tests/test_gpu_zz_pdl.py; LSD_PIPELINE_VG=0 / lsd_lio_set_pipeline turn it off).  Programmatic dependent launch stays
  // opt-in (LSD_PDL=1 / lsd_lio_set_pdl): it shortens the device time per scan, but cudaLaunchKernelEx costs the host more
  // per launch than a plain triple-chevron launch, and with a host loop that is synchronous per evaluation that is on the
  // critical path.
  { const char* ev = getenv("LSD_PDL"); l->pdl = (ev && ev[0] == '1') ? 1 : 0; }
  { const char* ev = getenv("LSD_PIPELINE_VG"); l->pipeline_vg = (ev && ev[0] == '0') ? 0 : 1; }
  // The reference's Nearest_Points rows outlive a search that finds nothing (laserMapping.cpp:1273, ivox3d.h:155-157);
  // reproducing that is what default-path parity needs (lsd_lio_set_stale_rows(l, 0) turns it off).
  l->stale_rows = true;
  // The neighbours reach esti_plane in the order IVox::GetClosestPoint returns them (DESIGN.md section 4: what takes the
  // posterior from ~4e-5 m to ~2e-7 m of laserMapping.cpp's); LSD_REF_ORDER=0 / lsd_lio_set_reference_order(l, 0) give the
  // faster sorted order instead.
  { const char* ev = getenv("LSD_REF_ORDER"); lsd_status_t r = lsd_lio_set_reference_order(l, (ev && ev[0] == '0') ? 0 : 1); if (r) { lsd_lio_destroy(l); return r; } }
  {  // cluster-shaped reuse evaluation: opt-in, LSD_REUSE_CLUSTER="CxT" = C CTAs of T threads.  The per-pass shuffle
     // reduction that keeps it inside 64 registers can cost more than the partials -> ticket -> last-block fold it replaces.
    const char* ev = getenv("LSD_REUSE_CLUSTER");
    l->reuse_cluster = (ev && ev[0] >= '1' && ev[0] <= '9') ? 1 : 0;
    int c = 0, t = 0;
    if (ev && sscanf(ev, "%dx%d", &c, &t) == 2 && c >= 1 && c <= 16 && t >= 32 && t <= 1024 && t % 32 == 0) { l->rc_ctas = c; l->rc_threads = t; }
#ifndef LSD_SIMT_EMU
    if (l->rc_ctas > 8) cudaFuncSetAttribute(lio_hmodel_reuse_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
#endif
  }
  *out = l;
  return LSD_OK;
}

lsd_status_t lsd_lio_destroy(lsd_lio_t* l) {
  if (!l) return LSD_OK;
  cudaSetDevice(l->device);
  if (l->stream) cudaStreamSynchronize(l->stream);
  if (l->copy_stream) { cudaStreamSynchronize(l->copy_stream); cudaStreamDestroy(l->copy_stream); }
  for (int i = 0; i < 2; i++) if (l->stage[i].ev) cudaEventDestroy(l->stage[i].ev);
  if (l->ev_main_vg) cudaEventDestroy(l->ev_main_vg);
  if (l->ev_side_vg) cudaEventDestroy(l->ev_side_vg);
  void* ptrs[] = {l->stage[0].buf, l->stage[1].buf, l->stage[0].body, l->stage[1].body, l->stage[0].dn, l->stage[1].dn, l->d_rows, l->d_body, l->d_n, l->d_near, l->d_near_cnt, l->d_selected, l->d_flags, l->d_plane, l->d_world,
                  l->d_partials, l->d_done, l->d_added, l->d_pabcd, l->d_plane_ok};
  for (void* p : ptrs) cudaFree(p);
  cudaFreeHost(l->h_result); cudaFreeHost(l->h_added);
  for (void* q : l->ipc_opened) cudaIpcCloseMemHandle(q);
  cudaFree(l->d_inbox); cudaFree(l->d_flagbox);
  cudaFree(l->d_ref_fallbacks);
  if (l->ev0) cudaEventDestroy(l->ev0);
  if (l->ev1) cudaEventDestroy(l->ev1);
  if (l->pev[0]) cudaEventDestroy(l->pev[0]);
  if (l->pev[1]) cudaEventDestroy(l->pev[1]);
  cudaStream_t own = l->stream;
  if (l->map) { if (l->map->stream == own) l->map->stream = nullptr; lsd_map_destroy(l->map); }
  if (l->vg) { if (l->vg->stream == own) l->vg->stream = nullptr; lsd_voxelgrid_destroy(l->vg); }
  if (own) cudaStreamDestroy(own);
  delete l;
  return LSD_OK;
}

lsd_map_t* lsd_lio_map(lsd_lio_t* l) { return l ? l->map : nullptr; }

lsd_status_t lsd_lio_set_stale_rows(lsd_lio_t* l, int flag) {
  if (!l) return LSD_ERR_INVALID;
  if (flag && l->map->view.shard_world > 1) { set_error("lsd_lio_set_stale_rows: not available on a tile-sharded handle"); return LSD_ERR_INVALID; }
  cudaSetDevice(l->device);
  // start from empty rows either way: a default-constructed Nearest_Points
  lio_clear_rows_kernel<<<(l->p.max_points + 255) / 256, 256, 0, l->stream>>>(l->d_near, l->d_near_cnt, l->p.max_points);
  LSD_CUDA(cudaMemsetAsync(l->d_rows, 0, 8, l->stream));
  LSD_CUDA(cudaStreamSynchronize(l->stream));
  l->stale_rows = flag != 0;
  l->rows_parity = 0;
  return LSD_OK;
}
// Neighbours in the reference's own order (warp_nth_element / rs_reference_order above).
lsd_status_t lsd_lio_set_reference_order(lsd_lio_t* l, int flag) {
  if (!l) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  if (flag && !l->d_ref_fallbacks) {
    LSD_CUDA(cudaMalloc((void**)&l->d_ref_fallbacks, 4));
    LSD_CUDA(cudaMemsetAsync(l->d_ref_fallbacks, 0, 4, l->stream));
    LSD_CUDA(cudaStreamSynchronize(l->stream));
  }
  l->reference_order = flag ? 1 : 0;
  return LSD_OK;
}
// Test entry: libstdc++'s std::nth_element(first, nth, last) as the search kernel replays it, on an arbitrary sequence of
// distances.  path_out: 1 = the warp-cooperative replay did it, 2 = it bailed out at introselect's depth limit and the serial
// replay took over (as in the kernel), 3 = serial replay (more than 32 elements).  perm_out[p] = index of the element at
// position p afterwards.  tests/test_gpu_lio.py compares it with the oracle's restatement, which is pinned to std::nth_element.
__global__ void __launch_bounds__(32) debug_nth_element_kernel(const float* __restrict__ dist, int n, int first, int nth, int last,
                                                               int* __restrict__ perm_out, int* __restrict__ path_out) {
  __shared__ unsigned char sr[kCandCap], six[kCandCap];
  const int lane = threadIdx.x & 31;
  int path = 3;
  if (n <= 32) {
    unsigned key = lane < n ? __float_as_uint(dist[lane]) : 0xffffffffu;
    int src = lane;
    path = 1;
    if (warp_nth_element(key, src, first, nth, last)) {
      if (lane < n) perm_out[lane] = src;
      if (lane == 0) *path_out = path;
      return;
    }
    path = 2;
  }
  for (int p = lane; p < n; p += 32) {
    int rk = 0;
    for (int t = 0; t < n; t++) rk += __float_as_uint(dist[t]) < __float_as_uint(dist[p]) ? 1 : 0;
    sr[p] = (unsigned char)rk; six[p] = (unsigned char)p;
  }
  __syncwarp();
  if (lane == 0) rs_nth_element(sr, six, first, nth, last);
  __syncwarp();
  for (int p = lane; p < n; p += 32) perm_out[p] = six[p];
  if (lane == 0) *path_out = path;
}
lsd_status_t lsd_debug_nth_element(const float* dist_host, int n, int first, int nth, int last, int* perm_out_host, int* path_out_host) {
  if (!dist_host || !perm_out_host || n < 0 || n > kCandCap || first < 0 || first > nth || nth > last || last > n) return LSD_ERR_INVALID;
  for (int i = 0; i < n; i++) if (!(dist_host[i] >= 0.f)) return LSD_ERR_INVALID;   // distances: non-negative, so that the bit patterns order like the values
  lsd_status_t s = ensure_device();
  if (s) return s;
  float* d = nullptr; int* o = nullptr;
  LSD_CUDA(cudaMalloc((void**)&d, (size_t)(n + 1) * 4));
  LSD_CUDA(cudaMalloc((void**)&o, (size_t)(n + 2) * 4));
  LSD_CUDA(cudaMemcpy(d, dist_host, (size_t)n * 4, cudaMemcpyHostToDevice));
  debug_nth_element_kernel<<<1, 32>>>(d, n, first, nth, last, o, o + n);
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(perm_out_host, o, (size_t)n * 4, cudaMemcpyDeviceToHost);
  int path = 0;
  if (e == cudaSuccess) e = cudaMemcpy(&path, o + n, 4, cudaMemcpyDeviceToHost);
  cudaFree(d); cudaFree(o);
  if (e != cudaSuccess) return cuda_fail(e, "lsd_debug_nth_element", __FILE__, __LINE__);
  if (path_out_host) *path_out_host = path;
  return LSD_OK;
}
// -> queries since the handle's creation whose candidates overflowed the search's list (answered in canonical order)
lsd_status_t lsd_lio_reference_order_fallbacks(lsd_lio_t* l, unsigned* count) {
  if (!l || !count) return LSD_ERR_INVALID;
  *count = 0;
  if (!l->d_ref_fallbacks) return LSD_OK;
  LSD_CUDA(cudaSetDevice(l->device));
  LSD_CUDA(cudaMemcpy(count, l->d_ref_fallbacks, 4, cudaMemcpyDeviceToHost));
  return LSD_OK;
}
// Programmatic dependent launch for the scan's kernel chain (lsd_common.cuh).  Off by default; LSD_PDL=1 in the
// environment turns it on at lsd_lio_create.  Results are bit-identical either way: only launch latency is hidden.
lsd_status_t lsd_lio_set_pdl(lsd_lio_t* l, int flag) {
  if (!l) return LSD_ERR_INVALID;
  l->pdl = flag ? 1 : 0;
  return LSD_OK;
}

// Pipelined voxel grid (lio.h): the downsample of a prefetched scan runs on the copy stream while the previous scan
// iterates.  Off by default; LSD_PIPELINE_VG=1 in the environment turns it on at lsd_lio_create.  Bit-identical results:
// the voxel grid is deterministic and reads nothing a scan computes.
lsd_status_t lsd_lio_set_pipeline(lsd_lio_t* l, int flag) {
  if (!l) return LSD_ERR_INVALID;
  l->pipeline_vg = flag ? 1 : 0;
  return LSD_OK;
}

lsd_status_t lsd_lio_pipeline_stats(lsd_lio_t* l, long long* issued, long long* adopted) {
  if (!l) return LSD_ERR_INVALID;
  if (issued) *issued = l->side_vg_issued;
  if (adopted) *adopted = l->side_vg_adopted;
  return LSD_OK;
}

lsd_status_t lsd_lio_set_knn_shape(lsd_lio_t* l, int shape) {
  if (!l || (shape != 0 && shape != 1)) return LSD_ERR_INVALID;
  l->knn_shape = shape;
  return LSD_OK;
}
lsd_status_t lsd_lio_set_nearby(lsd_lio_t* l, int stencil) {
  if (!l || (stencil != LSD_STENCIL_EXACT && stencil_slot(stencil) < 0)) return LSD_ERR_INVALID;
  l->p.ivox_nearby = stencil;
  return LSD_OK;
}
// Blob a rank publishes so the others can reach its inbox / flag box: same-process peers use the raw
// device pointers, other processes open the cudaIpc handles.
struct ShardBlob {
  long long pid;
  unsigned long long inbox, flagbox;
  cudaIpcMemHandle_t h_inbox, h_flagbox;
};
static_assert(sizeof(ShardBlob) <= LSD_SHARD_BLOB_BYTES, "LSD_SHARD_BLOB_BYTES too small");

lsd_status_t lsd_lio_shard_export(lsd_lio_t* l, int rank, int world, int tile_cells, int reach_cells, unsigned char* blob_out) {
  if (!l || !blob_out || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) { set_error("lsd_lio_shard_export: bad rank/world (max %d ranks)", kMaxRanks); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(l->device));
  lsd_status_t s = lsd_map_set_shard(l->map, rank, world, tile_cells, reach_cells);
  if (s) return s;
  if (!l->d_inbox) {
    LSD_CUDA(cudaMalloc((void**)&l->d_inbox, 2 * kInboxRegion * sizeof(double)));
    LSD_CUDA(cudaMemset(l->d_inbox, 0, 2 * kInboxRegion * sizeof(double)));
    const size_t fb = (size_t)l->p.max_points + kMaxRanks * sizeof(unsigned long long) + 64;
    LSD_CUDA(cudaMalloc((void**)&l->d_flagbox, fb));
    LSD_CUDA(cudaMemset(l->d_flagbox, 0, fb));
    LSD_CUDA(cudaDeviceSynchronize());
  }
  ShardBlob b;
  memset(&b, 0, sizeof(b));
  b.pid = (long long)getpid();
  b.inbox = (unsigned long long)l->d_inbox;
  b.flagbox = (unsigned long long)l->d_flagbox;
  LSD_CUDA(cudaIpcGetMemHandle(&b.h_inbox, l->d_inbox));
  LSD_CUDA(cudaIpcGetMemHandle(&b.h_flagbox, l->d_flagbox));
  memset(blob_out, 0, LSD_SHARD_BLOB_BYTES);
  memcpy(blob_out, &b, sizeof(b));
  l->shard_rank = rank; l->shard_world = world;
  if (world > 1) l->stale_rows = false;   // a non-owner rank has no row to keep (near_cnt = -1): documented deviation of the sharded mode
  return LSD_OK;
}

lsd_status_t lsd_lio_shard_connect(lsd_lio_t* l, const unsigned char* blobs) {
  if (!l || !blobs || l->shard_world < 1 || !l->d_inbox) { set_error("lsd_lio_shard_connect: call lsd_lio_shard_export first"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(l->device));
  ShardComm sc;
  memset(&sc, 0, sizeof(sc));
  sc.rank = l->shard_rank; sc.world = l->shard_world;
  for (int p = 0; p < sc.world; p++) {
    ShardBlob b;
    memcpy(&b, blobs + (size_t)p * LSD_SHARD_BLOB_BYTES, sizeof(b));
    if (p == sc.rank) { sc.inbox[p] = l->d_inbox; sc.flagbox[p] = l->d_flagbox; continue; }
    if (b.pid == (long long)getpid()) {  // peer handle in this process (possibly another device)
      sc.inbox[p] = reinterpret_cast<double*>(b.inbox);
      sc.flagbox[p] = reinterpret_cast<unsigned char*>(b.flagbox);
      cudaPointerAttributes at;
      if (cudaPointerGetAttributes(&at, sc.inbox[p]) == cudaSuccess && at.device != l->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return cuda_fail(e, "cudaDeviceEnablePeerAccess", __FILE__, __LINE__);
        cudaGetLastError();
      }
    } else {
      void *pi = nullptr, *pf = nullptr;
      LSD_CUDA(cudaIpcOpenMemHandle(&pi, b.h_inbox, cudaIpcMemLazyEnablePeerAccess));
      LSD_CUDA(cudaIpcOpenMemHandle(&pf, b.h_flagbox, cudaIpcMemLazyEnablePeerAccess));
      sc.inbox[p] = static_cast<double*>(pi);
      sc.flagbox[p] = static_cast<unsigned char*>(pf);
      l->ipc_opened.push_back(pi); l->ipc_opened.push_back(pf);
    }
  }
  l->sc = sc;
  l->seq = 0; l->mi_seq = 0;  // all ranks restart their sequence numbers together
  return LSD_OK;
}

// Tile-sharded handles: mean time one h-model evaluation spent in the in-kernel exchange (peer stores + waiting for the
// slowest peer's partial sums), in microseconds, and the number of evaluations averaged; resets the counters.
lsd_status_t lsd_lio_shard_exchange_stats(lsd_lio_t* l, double* mean_us, long long* evaluations) {
  if (!l || !mean_us) return LSD_ERR_INVALID;
  int khz = 0;
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, l->device);
  *mean_us = (l->xchg_count && khz > 0) ? l->xchg_cycles / (double)l->xchg_count / ((double)khz * 1e-3) : 0.0;
  if (evaluations) *evaluations = l->xchg_count;
  l->xchg_cycles = 0.0; l->xchg_count = 0;
  return LSD_OK;
}
lsd_status_t lsd_lio_sync(lsd_lio_t* l, double* gpu_ms_last, int* n_added_last) {
  if (!l) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  lsd_status_t s = lio_drain(l);
  if (s) return s;
  LSD_CUDA(cudaStreamSynchronize(l->stream));
  if (gpu_ms_last) *gpu_ms_last = l->last_gpu_ms;
  if (n_added_last) *n_added_last = l->last_added;
  return LSD_OK;
}
lsd_status_t lsd_lio_set_profile(lsd_lio_t* l, int on) {
  if (!l) return LSD_ERR_INVALID;
  l->profile = on ? 1 : 0;
  for (int k = 0; k < 4; k++) { l->prof_ms[k] = 0; l->prof_cnt[k] = 0; }
  return LSD_OK;
}
lsd_status_t lsd_lio_get_profile(lsd_lio_t* l, double* ms4, long long* cnt4) {
  if (!l || !ms4 || !cnt4) return LSD_ERR_INVALID;
  for (int k = 0; k < 4; k++) { ms4[k] = l->prof_ms[k]; cnt4[k] = l->prof_cnt[k]; }
  return LSD_OK;
}
lsd_status_t lsd_lio_set_next_id(lsd_lio_t* l, int32_t id) { if (!l) return LSD_ERR_INVALID; l->next_id = id; l->map_cells_known = 0; return LSD_OK; }
lsd_status_t lsd_lio_set_ekf_inited(lsd_lio_t* l, int flag) { if (!l) return LSD_ERR_INVALID; l->ekf_inited = flag ? 1 : 0; return LSD_OK; }

lsd_status_t lsd_lio_load_scan_dev(lsd_lio_t* l, const float* scan_dev, int n, int downsample, int* n_down) {
  if (!l || (n > 0 && !scan_dev)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  lsd_status_t s = lio_load(l, reinterpret_cast<const float4*>(scan_dev), n, downsample);
  if (s) return s;
  s = read_n_down(l);
  if (s) return s;
  if (n_down) *n_down = l->n_down;
  return LSD_OK;
}

lsd_status_t lsd_lio_load_scan(lsd_lio_t* l, const float* scan_host, int n, int downsample, int* n_down) {
  if (!l || (n > 0 && !scan_host)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  if (n > l->p.max_scan_points) { set_error("scan of %d points exceeds max_scan_points %d", n, l->p.max_scan_points); return LSD_ERR_CAPACITY; }
  lsd_lio::Stage* sg = free_stage(l);
  LSD_CUDA(cudaMemcpyAsync(sg->buf, scan_host, (size_t)n * 16, cudaMemcpyHostToDevice, l->stream));
  return lsd_lio_load_scan_dev(l, reinterpret_cast<const float*>(sg->buf), n, downsample, n_down);
}

lsd_status_t lsd_lio_get_down(lsd_lio_t* l, float* out_host, int cap, int* n_down) {
  if (!l || !out_host) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  if (l->n_down < 0) { lsd_status_t s = read_n_down(l); if (s) return s; }
  if (n_down) *n_down = l->n_down;
  const int c = std::min(cap, l->n_down);
  if (c > 0) LSD_CUDA(cudaMemcpyAsync(out_host, l->d_body, (size_t)c * 16, cudaMemcpyDeviceToHost, l->stream));
  LSD_CUDA(cudaStreamSynchronize(l->stream));
  return LSD_OK;
}

lsd_status_t lsd_lio_linearize(lsd_lio_t* l, const double* state26, int search, double* HTH36, double* HTh6, double* res_sum,
                               int* n_eff, int* degenerate) {
  if (!l || !state26 || !HTH36 || !HTh6 || !res_sum || !n_eff || !degenerate) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  return lio_linearize(l, state26, search != 0, HTH36, HTh6, res_sum, n_eff, degenerate);
}

lsd_status_t lsd_lio_get_matches(lsd_lio_t* l, int32_t* near_idx, float* near_xyz, int32_t* near_cnt, uint8_t* selected,
                                 float* plane, float* world) {
  if (!l || l->n_down < 0) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  const int n = l->n_down;
  cudaStream_t st = l->stream;
  std::vector<float4> nr;
  if (near_idx || near_xyz) { nr.resize((size_t)n * 5); LSD_CUDA(cudaMemcpyAsync(nr.data(), l->d_near, (size_t)n * 80, cudaMemcpyDeviceToHost, st)); }
  if (near_cnt) LSD_CUDA(cudaMemcpyAsync(near_cnt, l->d_near_cnt, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  if (selected) LSD_CUDA(cudaMemcpyAsync(selected, l->d_selected, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (plane) LSD_CUDA(cudaMemcpyAsync(plane, l->d_plane, (size_t)n * 16, cudaMemcpyDeviceToHost, st));
  if (world) LSD_CUDA(cudaMemcpyAsync(world, l->d_world, (size_t)n * 16, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  for (size_t i = 0; i < nr.size(); i++) {
    if (near_idx) memcpy(&near_idx[i], &nr[i].w, 4);
    if (near_xyz) { near_xyz[3 * i] = nr[i].x; near_xyz[3 * i + 1] = nr[i].y; near_xyz[3 * i + 2] = nr[i].z; }
  }
  return LSD_OK;
}

lsd_status_t lsd_lio_update(lsd_lio_t* l, double* state26_inout, double* P529_inout, lsd_lio_info_t* info) {
  if (!l || !state26_inout || !P529_inout) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  lsd_lio_info_t inf;
  memset(&inf, 0, sizeof(inf));
  const long long l0 = l->launches;
  lsd_status_t s = lio_update(l, state26_inout, P529_inout, &inf);
  inf.kernel_launches = (int)(l->launches - l0);
  if (info) *info = inf;
  return s;
}

lsd_status_t lsd_lio_map_incremental(lsd_lio_t* l, const double* state26, int* n_added) {
  if (!l || !state26) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  lsd_status_t s = lio_map_incremental(l, state26, 1, n_added, true);
  if (s == LSD_OK) l->map_cells_known = 1;
  return s;
}

static lsd_status_t prefetch_request(lsd_lio* l, const float* scan, int n, bool is_dev) {
  for (int i = 0; i < 2; i++)   // already staged (announced twice): one copy is enough, a second would outlive the scan that adopts the first
    if (l->stage[i].valid && l->stage[i].is_dev == is_dev && l->stage[i].host == scan && l->stage[i].n == n) return LSD_OK;
  if (l->stage[0].valid || l->stage[1].valid) {
    // a staged scan is waiting to be registered: that lsd_lio_scan call issues this copy (and voxel grid) once its first
    // kernels are in flight (issue_deferred_prefetch), so the driver calls do not delay it
    l->defer_host = scan; l->defer_n = n; l->defer_pending = true; l->defer_is_dev = is_dev;
    return LSD_OK;
  }
  // Every staging buffer is idle here: the voxel grid of the last scan (their only reader) finished before
  // lsd_lio_scan returned.
  l->defer_host = scan; l->defer_n = n; l->defer_pending = true; l->defer_is_dev = is_dev;
  return issue_deferred_prefetch(l);
}

lsd_status_t lsd_lio_prefetch(lsd_lio_t* l, const float* scan_host, int n) {
  if (!l || !scan_host || n <= 0) return LSD_ERR_INVALID;
  if (n > l->p.max_scan_points) { set_error("scan of %d points exceeds max_scan_points %d", n, l->p.max_scan_points); return LSD_ERR_CAPACITY; }
  LSD_CUDA(cudaSetDevice(l->device));
  return prefetch_request(l, scan_host, n, false);
}

lsd_status_t lsd_lio_prefetch_dev(lsd_lio_t* l, const float* scan_dev, int n) {
  if (!l || !scan_dev || n <= 0) return LSD_ERR_INVALID;
  if (n > l->p.max_scan_points) { set_error("scan of %d points exceeds max_scan_points %d", n, l->p.max_scan_points); return LSD_ERR_CAPACITY; }
  if (!l->pipeline_vg) return LSD_OK;   // nothing to copy: only the pipelined voxel grid has work to do ahead
  LSD_CUDA(cudaSetDevice(l->device));
  return prefetch_request(l, scan_dev, n, true);
}

lsd_status_t lsd_lio_scan_dev(lsd_lio_t* l, const float* scan_dev, int n, double* state26_inout, double* P529_inout,
                              lsd_lio_info_t* info) {
  if (!l || (n > 0 && !scan_dev) || !state26_inout || !P529_inout) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  l->pre = nullptr;
  if (l->defer_pending && l->defer_is_dev && l->defer_host == scan_dev && l->defer_n == n) l->defer_pending = false;  // requested, never issued
  for (int i = 0; i < 2; i++) {
    lsd_lio::Stage* sg = &l->stage[i];
    if (sg->valid && sg->is_dev && sg->host == scan_dev && sg->n == n) {   // downsampled ahead by lsd_lio_prefetch_dev
      LSD_CUDA(cudaStreamWaitEvent(l->stream, sg->ev, 0));
      sg->valid = false;
      l->pre = sg->down ? sg : nullptr;
    }
  }
  return lio_scan(l, reinterpret_cast<const float4*>(scan_dev), n, state26_inout, P529_inout, info);
}

lsd_status_t lsd_lio_scan(lsd_lio_t* l, const float* scan_host, int n, double* state26_inout, double* P529_inout,
                          lsd_lio_info_t* info) {
  if (!l || (n > 0 && !scan_host) || !state26_inout || !P529_inout) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(l->device));
  if (n > l->p.max_scan_points) { set_error("scan of %d points exceeds max_scan_points %d", n, l->p.max_scan_points); return LSD_ERR_CAPACITY; }
  lsd_lio::Stage* sg = nullptr;
  l->pre = nullptr;
  for (int i = 0; i < 2; i++) if (l->stage[i].valid && !l->stage[i].is_dev && l->stage[i].host == scan_host && l->stage[i].n == n) sg = &l->stage[i];
  if (l->defer_pending && !l->defer_is_dev && l->defer_host == scan_host && l->defer_n == n) l->defer_pending = false;  // requested, never issued: upload inline
  if (sg) {  // uploaded by lsd_lio_prefetch while the previous scan was being registered
    LSD_CUDA(cudaStreamWaitEvent(l->stream, sg->ev, 0));
    l->pre = sg->down ? sg : nullptr;   // also downsampled ahead (lsd_lio_set_pipeline)
  } else {
    sg = free_stage(l);
    sg->down = false; sg->is_dev = false;
    LSD_CUDA(cudaMemcpyAsync(sg->buf, scan_host, (size_t)n * 16, cudaMemcpyHostToDevice, l->stream));
  }
  sg->valid = false;
  l->busy_slot = (int)(sg - l->stage);
  const lsd_status_t rc = lio_scan(l, sg->buf, n, state26_inout, P529_inout, info);
  l->busy_slot = -1;
  return rc;
}

void lsd_lio_init_cov(double* P529) { if (P529) eskf::init_cov(P529); }
void lsd_state_boxplus(double* state26_inout, const double* delta23) { if (state26_inout && delta23) eskf::boxplus(state26_inout, delta23); }
void lsd_state_boxminus(const double* a26, const double* b26, double* out23) { if (a26 && b26 && out23) eskf::boxminus(a26, b26, out23); }

int lsd_eskf_update_table(double* state26_inout, double* P529_inout, const double* HTH36, const double* HTh6, const int* n_eff,
                          int n_table, double R, int max_iterations, double eps, int literal, int* converge_log16_or_null) {
  if (!state26_inout || !P529_inout || !HTH36 || !HTh6 || !n_eff || n_table < 1) return LSD_ERR_INVALID;
  int e = 0;
  auto hm = [&](const double*, bool converge, eskf::HModel* out) {
    if (converge_log16_or_null && e < 16) converge_log16_or_null[e] = converge ? 1 : 0;
    const int k = e < n_table ? e : n_table - 1;
    e++;
    out->n = n_eff[k];
    out->valid = n_eff[k] >= 1;
    if (!out->valid) return;
    memset(out->HTH, 0, sizeof(out->HTH)); memset(out->HTh, 0, sizeof(out->HTh));
    for (int a = 0; a < 6; a++) { for (int c = 0; c < 6; c++) out->HTH[15 * a + c] = HTH36[36 * k + 6 * a + c]; out->HTh[a] = HTh6[6 * k + a]; }
    if (out->n < eskf::N) { out->n = eskf::N; }  // the table form carries no h_x rows: small-n branch not exercised here
  };
  eskf::UpdateResult r = eskf::update_iterated(state26_inout, P529_inout, hm, R, max_iterations, eps, literal != 0);
  return r.evaluations;
}

}  // extern "C"
