// reg.cu — scan matcher behind the pcl::Registration-shaped seam: NDT (P2D, DIRECT1/7/27) and
// GICP (D2D), Levenberg-Marquardt on SE(3), fitness score.
//
// Replaces (reference: slam/thirdparty/fast_gicp):
//   LsqRegistration::computeTransformation / step_lm / is_converged
//                              include/fast_gicp/gicp/impl/lsq_registration_impl.hpp:71-131,163-208
//   se3_exp (rotation first)   include/fast_gicp/so3/so3.hpp:80-104
//   NDTCudaCore + kernels      src/fast_gicp/cuda/{ndt_cuda,gaussian_voxelmap,find_voxel_correspondences,
//                              ndt_compute_derivatives,covariance_regularization}.cu
//   FastGICP                   include/fast_gicp/gicp/impl/fast_gicp_impl.hpp:119-303
//   getFitnessScore            pcl::Registration (PCL 1.9.1), call sites loop_detector.hpp:180,206
// Differences in shape, not in result:
//   * The reference NDT launches one thrust transform per neighbour offset, compacts the pair list with
//     remove_if and reduces 172-byte fp32 tuples; here one kernel per cost evaluation looks the
//     offsets up, evaluates and reduces (double accumulators, fixed order).
//   * PLANE-regularised covariances are V diag(1e-3,1,1) V^T (NDT) / U diag(1,1,1e-3) V^T (GICP):
//     C = I - 0.999 n n^T with n the smallest-eigenvalue direction.  Only n is stored (12 bytes instead
//     of 36/128), C^-1 = I + 999 n n^T is applied in closed form, no per-correspondence 3x3 inversion
//     for NDT.
//   * GICP neighbours come from the hash-voxel map's exact search (knn.cuh) instead of a k-d tree.
#include <unistd.h>

#include <cfloat>
#include <chrono>
#include <type_traits>
#include <vector>

#include "knn.cuh"
#include "lio.h"
#include "map.h"

namespace lsd {

// ------------------------------------------------------------------ NDT voxel table
struct __align__(128) NdtBuildLine { unsigned long long key; unsigned count; unsigned pad; double sum[3]; double sxx[6]; };
struct __align__(64) NdtLine { unsigned long long key; int n; float mean[3]; float nrm[3]; float pad[7]; };
static_assert(sizeof(NdtLine) == 64, "NdtLine must be two sectors");

struct NdtView { NdtLine* lines; unsigned long long mask; float res; };

// calc_voxel_coord, vector3_hash.cuh:35-38
__device__ __forceinline__ int3 ndt_coord(float x, float y, float z, float res) {
  return make_int3((int)floorf(x / res - 0.5f), (int)floorf(y / res - 0.5f), (int)floorf(z / res - 0.5f));
}

// The build-table slot of voxel `key` (open addressing, linear probing), claimed if the voxel is new; -1 when kMaxProbe
// probes find neither the key nor a free slot.  Both voxel maps (NDT, VGICP) are accumulated through here.
__device__ __forceinline__ long long claim_slot(NdtBuildLine* __restrict__ tab, unsigned long long mask, unsigned long long key) {
  unsigned long long s = hash_key(key) & mask;
  for (unsigned probe = 0; probe < kMaxProbe; probe++) {
    unsigned long long* kp = &tab[s].key;
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(kp);
    if (cur == 0ull) cur = atomicCAS(kp, 0ull, key), cur = cur == 0ull ? key : cur;
    if (cur == key) return (long long)s;
    s = (s + 1) & mask;
  }
  return -1;
}

// Tile-sharded target (SURVEY.md section 8e, row C3): with world > 1 a rank keeps only the voxels of the x-y tiles it owns
// (tile_owner, lsd_common.cuh).  Every (source point, stencil offset) pair then finds its voxel on exactly one rank, so the
// ranks' sums partition the single-GPU sums and the in-kernel all-reduce (grid_finalize) restores them: no halo needed.
__global__ void __launch_bounds__(256) ndt_accum_kernel(NdtBuildLine* __restrict__ tab, unsigned long long mask, float res,
                                                        const float4* __restrict__ pts, int n, unsigned* __restrict__ fail,
                                                        int shard_rank, int shard_world, int shard_tile) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = __ldg(pts + i);
  const int3 c = ndt_coord(p.x, p.y, p.z, res);
  if (!coord_ok(c.x, c.y, c.z)) { atomicAdd(fail, 1u); return; }
  if (shard_world > 1 && tile_owner(c.x, c.y, shard_tile, shard_world) != shard_rank) return;   // another rank's voxel
  const long long s = claim_slot(tab, mask, pack_key(c.x, c.y, c.z, 0));
  if (s < 0) { atomicAdd(fail, 1u); return; }
  atomicAdd(&tab[s].count, 1u);
  const double x = p.x, y = p.y, z = p.z;
  atomicAdd(&tab[s].sum[0], x); atomicAdd(&tab[s].sum[1], y); atomicAdd(&tab[s].sum[2], z);
  atomicAdd(&tab[s].sxx[0], x * x); atomicAdd(&tab[s].sxx[1], x * y); atomicAdd(&tab[s].sxx[2], x * z);
  atomicAdd(&tab[s].sxx[3], y * y); atomicAdd(&tab[s].sxx[4], y * z); atomicAdd(&tab[s].sxx[5], z * z);
}

// smallest-eigenvalue direction of a symmetric 3x3 (double, cyclic Jacobi)
__host__ __device__ inline void smallest_eigvec(const double* Ain, double* nrm) {
  double A[9], V[9];
  for (int i = 0; i < 9; i++) { A[i] = Ain[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 30; sweep++) {
    if (fabs(A[1]) + fabs(A[2]) + fabs(A[5]) <= 1e-18 * (fabs(A[0]) + fabs(A[4]) + fabs(A[8])) + 1e-300) break;
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
  int k0 = 0;
  if (A[4] < A[0]) k0 = 1;
  if (A[8] < A[4 * k0]) k0 = 2;
  nrm[0] = V[k0]; nrm[1] = V[3 + k0]; nrm[2] = V[6 + k0];
}

// ndt_finalize_voxels_kernel (gaussian_voxelmap.cu:181-202) + PLANE regularisation
__global__ void __launch_bounds__(256) ndt_finalize_kernel(const NdtBuildLine* __restrict__ tab, NdtLine* __restrict__ out,
                                                           unsigned long long n_lines, unsigned* __restrict__ n_vox) {
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_lines) return;
  NdtLine o;
  o.key = tab[s].key; o.n = 0;
  for (int k = 0; k < 3; k++) { o.mean[k] = 0.f; o.nrm[k] = 0.f; }
  for (int k = 0; k < 7; k++) o.pad[k] = 0.f;
  if (o.key != 0ull) {
    const double n = (double)tab[s].count;
    const double* S = tab[s].sum; const double* X = tab[s].sxx;
    const double m[3] = {S[0] / n, S[1] / n, S[2] / n};
    double C[9];
    C[0] = (X[0] - m[0] * S[0]) / n; C[1] = (X[1] - m[0] * S[1]) / n; C[2] = (X[2] - m[0] * S[2]) / n;
    C[4] = (X[3] - m[1] * S[1]) / n; C[5] = (X[4] - m[1] * S[2]) / n; C[8] = (X[5] - m[2] * S[2]) / n;
    C[3] = C[1]; C[6] = C[2]; C[7] = C[5];
    double nr[3];
    smallest_eigvec(C, nr);
    o.n = (int)tab[s].count;
    for (int k = 0; k < 3; k++) { o.mean[k] = (float)m[k]; o.nrm[k] = (float)nr[k]; }
    atomicAdd(n_vox, 1u);
  }
  out[s] = o;
}

// Slot of voxel (x, y, z) in a finalised voxel table (NdtView, VgView), -1 if absent.
template <class View>
__device__ __forceinline__ int voxel_lookup(const View& v, int x, int y, int z) {
  if (!coord_ok(x, y, z)) return -1;
  const unsigned long long key = pack_key(x, y, z, 0);
  unsigned long long s = hash_key(key) & v.mask;
  for (unsigned probe = 0; probe < kMaxProbe; probe++) {
    const unsigned long long k = __ldg(&v.lines[s].key);
    if (k == key) return (int)s;
    if (k == 0ull) return -1;
    s = (s + 1) & v.mask;
  }
  return -1;
}

// Offset o of the DIRECT1 / DIRECT7 / DIRECT27 neighbour stencil (n_off = 1, 7, 27)
__constant__ signed char c_ndt_off7[7][3] = {{0,0,0},{1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1}};
__device__ __forceinline__ int3 stencil_offset(int o, int n_off) {
  if (n_off == 27) return make_int3(o / 9 - 1, (o / 3) % 3 - 1, o % 3 - 1);
  return make_int3(c_ndt_off7[o][0], c_ndt_off7[o][1], c_ndt_off7[o][2]);
}

struct Pose34f { float R[9], t[3]; };
struct Pose34d { double R[9], t[3]; };

// R a + t
__device__ __forceinline__ float3 xform(const Pose34f& T, const float4 a) {
  return make_float3(T.R[0] * a.x + T.R[1] * a.y + T.R[2] * a.z + T.t[0], T.R[3] * a.x + T.R[4] * a.y + T.R[5] * a.z + T.t[1],
                     T.R[6] * a.x + T.R[7] * a.y + T.R[8] * a.z + T.t[2]);
}
__device__ __forceinline__ double3 xform(const Pose34d& T, const float4 a) {
  const double ax = a.x, ay = a.y, az = a.z;
  return make_double3(T.R[0] * ax + T.R[1] * ay + T.R[2] * az + T.t[0], T.R[3] * ax + T.R[4] * ay + T.R[5] * az + T.t[1],
                      T.R[6] * ax + T.R[7] * ay + T.R[8] * az + T.t[2]);
}

// One source point of an NDT cost evaluation (find_voxel_correspondences + p2d_ndt_compute_derivatives).  `corr` points at
// the [n_off, n] correspondence slots of this cloud.  Shared by the single-pair kernel below (compile-time flags) and the
// batched loop-closure kernel (loop.cu, flags per candidate): the same expressions, so the same bits.
__device__ __forceinline__ void ndt_point(const NdtView& v, const float4 a, int i, int n, int n_off, const Pose34f& lin,
                                          const Pose34f& ev, int* __restrict__ corr, bool update, bool deriv, double (&vals)[29]) {
  const float k_sq = v.res * v.res;
  const float3 t = xform(ev, a);
  const float tx = t.x, ty = t.y, tz = t.z;
  int3 c = make_int3(0, 0, 0);
  if (update) {
    const float3 l = xform(lin, a);
    c = ndt_coord(l.x, l.y, l.z, v.res);
  }
#pragma unroll 1
  for (int o = 0; o < n_off; o++) {
    int slot;
    if (update) {
      const int3 d = stencil_offset(o, n_off);
      slot = voxel_lookup(v, c.x + d.x, c.y + d.y, c.z + d.z);
      corr[(size_t)o * n + i] = slot;
    } else {
      slot = corr[(size_t)o * n + i];
    }
    if (slot < 0) continue;
    vals[28] += 1.0;  // correspondences found
    const NdtLine* ln = v.lines + slot;
    const float4 h = __ldg(reinterpret_cast<const float4*>(ln) + 0);          // key lo/hi, n, mean.x
    const float4 g = __ldg(reinterpret_cast<const float4*>(ln) + 1);          // mean.y, mean.z, nrm.x, nrm.y
    const float nz = __ldg(reinterpret_cast<const float*>(ln) + 8);
    if (__float_as_int(h.z) <= 6) continue;                                   // ndt_compute_derivatives.cu:62-64
    const float mx = h.w, my = g.x, mz = g.y, nx = g.z, ny = g.w;
    const float ex = mx - tx, ey = my - ty, ez = mz - tz;
    const float ne = nx * ex + ny * ey + nz * ez;
    const float cx = ex + 999.0f * nx * ne, cy = ey + 999.0f * ny * ne, cz = ez + 999.0f * nz * ne;  // C^-1 e
    const float xn = sqrtf(ex * ex + ey * ey + ez * ez);
    const float w = k_sq / (k_sq + xn * xn);                                   // cauchy
    vals[27] += (double)(w * (ex * cx + ey * cy + ez * cz));
    if (deriv) {
      const float J[3][6] = {{0.f, -tz, ty, -1.f, 0.f, 0.f}, {tz, 0.f, -tx, 0.f, -1.f, 0.f}, {-ty, tx, 0.f, 0.f, 0.f, -1.f}};
      float M[3][6];
#pragma unroll
      for (int cc = 0; cc < 6; cc++) {
        const float nj = nx * J[0][cc] + ny * J[1][cc] + nz * J[2][cc];
        M[0][cc] = J[0][cc] + 999.0f * nx * nj; M[1][cc] = J[1][cc] + 999.0f * ny * nj; M[2][cc] = J[2][cc] + 999.0f * nz * nj;
      }
      int q = 0;
#pragma unroll
      for (int p = 0; p < 6; p++) {
#pragma unroll
        for (int r = p; r < 6; r++) vals[q++] += (double)(w * (J[0][p] * M[0][r] + J[1][p] * M[1][r] + J[2][p] * M[2][r]));
        vals[21 + p] += (double)(w * (J[0][p] * cx + J[1][p] * cy + J[2][p] * cz));
      }
    }
  }
}

// One NDT cost evaluation (find_voxel_correspondences + p2d_ndt_compute_derivatives + sum).
// UPDATE: look the correspondences up at the linearisation pose and store them; else reuse.
// DERIV: accumulate H (21) and b (6) besides the error.
template <bool UPDATE, bool DERIV>
__global__ void __launch_bounds__(256) ndt_cost_kernel(NdtView v, const float4* __restrict__ src, int n, int n_off, Pose34f lin,
                                                       Pose34f ev, int* __restrict__ corr, double* __restrict__ partials,
                                                       unsigned* __restrict__ done, double* __restrict__ result, double seq,
                                                       ShardComm sc) {
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    ndt_point(v, __ldg(src + i), i, n, n_off, lin, ev, corr, UPDATE, DERIV, vals);
  block_partials<29>(vals, partials);
  grid_finalize<29>(partials, done, result, 0, -1, 0.0, kResSeq, seq, sc, 0);
}

// ------------------------------------------------------------------ GICP
// k-NN covariance -> smallest-eigenvalue direction (calculate_covariances, fast_gicp_impl.hpp:244-303).
// One warp per point: exact K-NN, lanes hold the neighbours, warp-shuffle moments in double.
constexpr int kRegWarps = 8;

// Lanes 0 .. k-1 hold the k neighbours (x, y, z; zero in lanes without one): the k-column mean and covariance, its
// smallest-eigenvalue direction, stored by lane 0 with nf, the neighbour count, into nrm[4 i .. 4 i + 4).
__device__ __forceinline__ void warp_normal(double x, double y, double z, int k, int nf, double* __restrict__ nrm, int i) {
  const int lane = threadIdx.x & 31;
  const double kk = (double)k;
  const double mx = warp_sum(x) / kk, my = warp_sum(y) / kk, mz = warp_sum(z) / kk;   // rowwise().mean() over k columns
  const double dx = (lane < k ? x : 0.0) - (lane < k ? mx : 0.0), dy = (lane < k ? y : 0.0) - (lane < k ? my : 0.0),
               dz = (lane < k ? z : 0.0) - (lane < k ? mz : 0.0);
  double C[9];
  C[0] = warp_sum(dx * dx) / kk; C[1] = warp_sum(dx * dy) / kk; C[2] = warp_sum(dx * dz) / kk;
  C[4] = warp_sum(dy * dy) / kk; C[5] = warp_sum(dy * dz) / kk; C[8] = warp_sum(dz * dz) / kk;
  C[3] = C[1]; C[6] = C[2]; C[7] = C[5];
  if (lane == 0) {
    double nr[3];
    smallest_eigvec(C, nr);
    double* o = nrm + 4 * (size_t)i;  // double: C = I - 0.999 n n^T is inverted with condition number 1000
    o[0] = nr[0]; o[1] = nr[1]; o[2] = nr[2]; o[3] = (double)nf;
  }
}

__global__ void __launch_bounds__(kRegWarps * 32, 3) gicp_normals_kernel(MapView mv, const float4* __restrict__ pts, int n, int k,
                                                                         float max_sq, double* __restrict__ nrm) {
  __shared__ __align__(16) unsigned char s_list[kRegWarps * kWarpListBytes];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpList wl = make_warp_list(s_list, warp);
  for (int i = blockIdx.x * kRegWarps + warp; i < n; i += gridDim.x * kRegWarps) {
    const float4 p = __ldg(pts + i);
    Neighbor nb;
    const int nf = knn_exact_warp<20>(mv, p.x, p.y, p.z, max_sq, wl, nb);
    double x = 0, y = 0, z = 0;
    if (lane < min(nf, k)) { const float4 q = load_loc(mv, nb.loc); x = q.x; y = q.y; z = q.z; }
    warp_normal(x, y, z, k, nf, nrm, i);
  }
}

// The reference takes the k nearest neighbours wherever they are (pcl::search::KdTree::nearestKSearch,
// fast_gicp_impl.hpp:259); max_sq above only bounds the fast grid search.  Points that found fewer than k inside the
// radius — sparse rings of a scan at long range — are completed here by an exact scan of the whole cloud: one warp per
// such point, the k best kept sorted across lanes 0 .. k-1 in registers (insert = ballot rank + one shuffle).
__global__ void __launch_bounds__(kRegWarps * 32) gicp_normals_complete_kernel(const float4* __restrict__ pts, int n, int k,
                                                                              double* __restrict__ nrm) {
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * kRegWarps + (threadIdx.x >> 5); i < n; i += gridDim.x * kRegWarps) {
    if (nrm[4 * (size_t)i + 3] >= (double)k) continue;     // warp-uniform
    const float4 p = __ldg(pts + i);
    float bd = 3.0e38f; int bi = 0x7fffffff;               // lane r: r-th best so far (lanes >= k unused)
    for (int j0 = 0; j0 < n; j0 += 32) {
      const int j = j0 + lane;
      float d2 = 3.0e38f;
      if (j < n) { const float4 a = __ldg(pts + j); d2 = dist2(p.x, p.y, p.z, a.x, a.y, a.z); }
      // worst kept entry (lane k-1) as the admission test
      const float wd = __shfl_sync(0xffffffffu, bd, k - 1); const int wi = __shfl_sync(0xffffffffu, bi, k - 1);
      unsigned cand = __ballot_sync(0xffffffffu, j < n && (d2 < wd || (d2 == wd && j < wi)));
      while (cand) {
        const int src = __ffs(cand) - 1;
        cand &= cand - 1;
        const float nd = __shfl_sync(0xffffffffu, d2, src); const int ni = j0 + src;
        const bool less = bd < nd || (bd == nd && bi < ni);                 // my entry stays before the new one
        const int pos = __popc(__ballot_sync(0xffffffffu, less && lane < k));
        const float ud = __shfl_up_sync(0xffffffffu, bd, 1); const int ui = __shfl_up_sync(0xffffffffu, bi, 1);
        if (pos < k) {
          if (lane == pos) { bd = nd; bi = ni; }
          else if (lane > pos && lane < k) { bd = ud; bi = ui; }
        }
      }
    }
    const int nf = min(n, k);
    double x = 0, y = 0, z = 0;
    if (lane < nf) { const float4 q = __ldg(pts + bi); x = q.x; y = q.y; z = q.z; }
    warp_normal(x, y, z, k, nf, nrm, i);
  }
}

// Exact nearest neighbour with d2 <= max_sq for ONE THREAD (batched shape, cf. knn_query_thread_kernel): Chebyshev
// shells around the query's voxel, tag probes in L2, cells pruned by their distance to the query, stop as soon as
// no unseen shell can hold a closer point.  Same result as knn_exact_warp<1> (any exact search gives the same
// (d2, id) minimum).
__device__ __forceinline__ bool nn1_exact_thread(const MapView& mv, float qx, float qy, float qz, float max_sq, float* d2_out,
                                                 int* id_out) {
  const int3 c = pos2grid(qx, qy, qz, mv.inv_res);
  const float fx = qx * mv.inv_res - (float)c.x, fy = qy * mv.inv_res - (float)c.y, fz = qz * mv.inv_res - (float)c.z;
  const int rmax = (int)ceilf(sqrtf(max_sq) * mv.inv_res) + 1;
  float bd = 3.0e38f; int bi = 0x7fffffff;
  bool found = false;
  const float res2 = mv.res * mv.res * (1.0f - 4e-5f);
  for (int r = 0; r <= rmax; r++) {
    const float bound = found ? bd : max_sq;
    if (r >= 1) { const float lo = (float)(r - 1); if (bound < lo * lo * res2) break; }
    for (int i = -r; i <= r; i++) {
      const float gx = fmaxf(0.f, fmaxf((float)i - 0.5f - fx, fx - ((float)i + 0.5f)));
      for (int j = -r; j <= r; j++) {
        const float gy = fmaxf(0.f, fmaxf((float)j - 0.5f - fy, fy - ((float)j + 0.5f)));
        const bool face = (i == -r || i == r || j == -r || j == r);
        const int step = face ? 1 : max(2 * r, 1);
        for (int l = -r; l <= r; l += step) {
          const float gz = fmaxf(0.f, fmaxf((float)l - 0.5f - fz, fz - ((float)l + 0.5f)));
          const float cur = found ? bd : max_sq;
          if ((gx * gx + gy * gy + gz * gz) * res2 > cur) continue;  // no point of this voxel can beat the current best
          const int x = c.x + i, y = c.y + j, z = c.z + l;
          if (!coord_ok(x, y, z)) continue;
          const unsigned long long key = pack_key(x, y, z, 0);
          uint4 h;
          const CellLine* ln = tag_find(mv, key, &h);
          if (!ln) continue;
          const unsigned cnt = h.z;
          const int levels = cnt > (unsigned)kPtsPerLine ? min((int)((cnt - 1) / kPtsPerLine), kMaxLevel) : 0;
          for (int L = 0; L <= levels; L++) {
            const CellLine* ll = ln;
            if (L > 0) { uint4 hl; ll = tag_find(mv, key | ((unsigned long long)L << 57), &hl); if (!ll) continue; }
            const int n = (int)min(cnt - (unsigned)(L * kPtsPerLine), (unsigned)kPtsPerLine);
            for (int k = 0; k < n; k++) {
              const float4 a = ldg_f4(&ll->pts[k]);
              const float d2 = dist2(qx, qy, qz, a.x, a.y, a.z);
              const int pid = __float_as_int(a.w);
              if (d2 <= max_sq && (d2 < bd || (d2 == bd && pid < bi))) { bd = d2; bi = pid; found = true; }
            }
          }
        }
      }
    }
  }
  *d2_out = bd; *id_out = bi;
  return found;
}

// Mahalanobis matrix (C_B + R C_A R^T)^-1 of correspondence (source i, target c) at T, in double, stored symmetric
// (xx xy xz yy yz zz) into maha[6 i ..].
__device__ __forceinline__ void gicp_store_maha(const double* __restrict__ src_nrm, const double* __restrict__ tgt_nrm, int i, int c,
                                                const Pose34d& T, double* __restrict__ maha) {
  const double* na = src_nrm + 4 * (size_t)i;
  const double* nbv = tgt_nrm + 4 * (size_t)c;
  const double rn[3] = {T.R[0] * na[0] + T.R[1] * na[1] + T.R[2] * na[2], T.R[3] * na[0] + T.R[4] * na[1] + T.R[5] * na[2],
                        T.R[6] * na[0] + T.R[7] * na[1] + T.R[8] * na[2]};
  double A[9];
#pragma unroll
  for (int p = 0; p < 3; p++)
#pragma unroll
    for (int q = 0; q < 3; q++) A[3 * p + q] = (p == q ? 2.0 : 0.0) - 0.999 * (nbv[p] * nbv[q] + rn[p] * rn[q]);
  const double c00 = A[4] * A[8] - A[5] * A[7], c01 = A[5] * A[6] - A[3] * A[8], c02 = A[3] * A[7] - A[4] * A[6];
  const double idet = 1.0 / (A[0] * c00 + A[1] * c01 + A[2] * c02);
  double* M = maha + 6 * (size_t)i;
  M[0] = c00 * idet; M[1] = (A[2] * A[7] - A[1] * A[8]) * idet; M[2] = (A[1] * A[5] - A[2] * A[4]) * idet;
  M[3] = (A[0] * A[8] - A[2] * A[6]) * idet; M[4] = (A[2] * A[3] - A[0] * A[5]) * idet; M[5] = (A[0] * A[4] - A[1] * A[3]) * idet;
}

// update_correspondences (fast_gicp_impl.hpp:119-157): 1-NN of the transformed source point, Mahalanobis
// matrix.  One warp per source point.
__global__ void __launch_bounds__(kRegWarps * 32, 3) gicp_corr_kernel(MapView mv, const float4* __restrict__ src,
                                                                      const double* __restrict__ src_nrm, int n,
                                                                      const double* __restrict__ tgt_nrm, Pose34d T, Pose34f Tf,
                                                                      float max_corr_sq, int* __restrict__ corr,
                                                                      double* __restrict__ maha) {
  __shared__ __align__(16) unsigned char s_list[kRegWarps * kWarpListBytes];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpList wl = make_warp_list(s_list, warp);
  for (int i = blockIdx.x * kRegWarps + warp; i < n; i += gridDim.x * kRegWarps) {
    const float3 q = xform(Tf, __ldg(src + i));
    Neighbor nb;
    const int nf = knn_exact_warp<1>(mv, q.x, q.y, q.z, max_corr_sq, wl, nb);
    const float d2 = __shfl_sync(kFull, nb.d2, 0);
    const int id = __shfl_sync(kFull, nb.id, 0);
    if (lane != 0) continue;
    const int c = (nf > 0 && d2 < max_corr_sq) ? id : -1;
    corr[i] = c;
    if (c >= 0) gicp_store_maha(src_nrm, tgt_nrm, i, c, T, maha);
  }
}

// update_correspondences, batched shape: one thread per source point (nn1_exact_thread)
__global__ void __launch_bounds__(256) gicp_corr_thread_kernel(MapView mv, const float4* __restrict__ src, const double* __restrict__ src_nrm,
                                                               int n, const double* __restrict__ tgt_nrm, Pose34d T, Pose34f Tf,
                                                               float max_corr_sq, int* __restrict__ corr, double* __restrict__ maha) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float3 q = xform(Tf, __ldg(src + i));
  float d2; int id;
  const bool f = nn1_exact_thread(mv, q.x, q.y, q.z, max_corr_sq, &d2, &id);
  const int c = (f && d2 < max_corr_sq) ? id : -1;
  corr[i] = c;
  if (c >= 0) gicp_store_maha(src_nrm, tgt_nrm, i, c, T, maha);
}

// One distribution-to-distribution residual e at the transformed point t with Mahalanobis matrix M, weighted by w:
// e^T M e into vals[27] and, with deriv, J^T M J (upper triangle) into vals[0..21) and J^T M e into vals[21..27), with
// J = d(t)/d(rotation, translation).  GICP passes w = 1.0 (an exact product), VGICP sqrt(voxel points).
__device__ __forceinline__ void accum_d2d(double (&vals)[29], const double (&M)[3][3], const double3 e, const double3 t, double w,
                                          bool deriv) {
  const double cx = M[0][0] * e.x + M[0][1] * e.y + M[0][2] * e.z, cy = M[1][0] * e.x + M[1][1] * e.y + M[1][2] * e.z,
               cz = M[2][0] * e.x + M[2][1] * e.y + M[2][2] * e.z;
  vals[27] += w * (e.x * cx + e.y * cy + e.z * cz);
  if (deriv) {
    const double J[3][6] = {{0., -t.z, t.y, -1., 0., 0.}, {t.z, 0., -t.x, 0., -1., 0.}, {-t.y, t.x, 0., 0., 0., -1.}};
    double MJ[3][6];
#pragma unroll
    for (int cc = 0; cc < 6; cc++) {
      MJ[0][cc] = M[0][0] * J[0][cc] + M[0][1] * J[1][cc] + M[0][2] * J[2][cc];
      MJ[1][cc] = M[1][0] * J[0][cc] + M[1][1] * J[1][cc] + M[1][2] * J[2][cc];
      MJ[2][cc] = M[2][0] * J[0][cc] + M[2][1] * J[1][cc] + M[2][2] * J[2][cc];
    }
    int q = 0;
#pragma unroll
    for (int p = 0; p < 6; p++) {
#pragma unroll
      for (int r = p; r < 6; r++) vals[q++] += w * (J[0][p] * MJ[0][r] + J[1][p] * MJ[1][r] + J[2][p] * MJ[2][r]);
      vals[21 + p] += w * (J[0][p] * cx + J[1][p] * cy + J[2][p] * cz);
    }
  }
}

// linearize / compute_error (fast_gicp_impl.hpp:159-242), one thread per source point, double.
template <bool DERIV>
__global__ void __launch_bounds__(256) gicp_cost_kernel(const float4* __restrict__ src, int n, const float4* __restrict__ tgt,
                                                        Pose34d T, const int* __restrict__ corr, const double* __restrict__ maha,
                                                        double* __restrict__ partials, unsigned* __restrict__ done,
                                                        double* __restrict__ result, double seq, ShardComm sc) {
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int c = corr[i];
    if (c < 0) continue;
    vals[28] += 1.0;
    const float4 b = __ldg(tgt + c);
    const double3 t = xform(T, __ldg(src + i));
    const double3 e = make_double3((double)b.x - t.x, (double)b.y - t.y, (double)b.z - t.z);
    const double* Ms = maha + 6 * (size_t)i;
    const double M[3][3] = {{Ms[0], Ms[1], Ms[2]}, {Ms[1], Ms[3], Ms[4]}, {Ms[2], Ms[4], Ms[5]}};
    accum_d2d(vals, M, e, t, 1.0, DERIV);
  }
  block_partials<29>(vals, partials);
  grid_finalize<29>(partials, done, result, 0, -1, 0.0, kResSeq, seq, sc, 0);
}

// ------------------------------------------------------------------ VGICP
// FastVGICP (fast_vgicp_impl.hpp:72-207) on a GaussianVoxelMap with ADDITIVE voxels
// (fast_vgicp_voxel.hpp:108-182): voxel = mean of its points and MEAN of their PLANE-regularised
// covariances I - 0.999 n n^T; coord = floor(x/res - 0.5) in double; weight sqrt(num_points).
struct __align__(128) VgLine { unsigned long long key; int n; int pad; double mean[3]; double cov[6]; double pad2[4]; };
static_assert(sizeof(VgLine) == 128, "VgLine must be one line");
struct VgView { VgLine* lines; unsigned long long mask; double res; };

__device__ __forceinline__ int3 vg_coord(double x, double y, double z, double res) {
  return make_int3((int)floor(x / res - 0.5), (int)floor(y / res - 0.5), (int)floor(z / res - 0.5));
}

// GaussianVoxelMap::create_voxelmap: sum[] = sum of points, sxx[] = sum of covariances (xx xy xz yy yz zz)
__global__ void __launch_bounds__(256) vgicp_accum_kernel(NdtBuildLine* __restrict__ tab, unsigned long long mask, double res,
                                                          const float4* __restrict__ pts, const double* __restrict__ nrm, int n,
                                                          unsigned* __restrict__ fail) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = __ldg(pts + i);
  const double x = p.x, y = p.y, z = p.z;
  const int3 c = vg_coord(x, y, z, res);
  if (!coord_ok(c.x, c.y, c.z)) { atomicAdd(fail, 1u); return; }
  const long long s = claim_slot(tab, mask, pack_key(c.x, c.y, c.z, 0));
  if (s < 0) { atomicAdd(fail, 1u); return; }
  const double nx = nrm[4 * (size_t)i], ny = nrm[4 * (size_t)i + 1], nz = nrm[4 * (size_t)i + 2];
  atomicAdd(&tab[s].count, 1u);
  atomicAdd(&tab[s].sum[0], x); atomicAdd(&tab[s].sum[1], y); atomicAdd(&tab[s].sum[2], z);
  atomicAdd(&tab[s].sxx[0], 1.0 - 0.999 * nx * nx); atomicAdd(&tab[s].sxx[1], -0.999 * nx * ny); atomicAdd(&tab[s].sxx[2], -0.999 * nx * nz);
  atomicAdd(&tab[s].sxx[3], 1.0 - 0.999 * ny * ny); atomicAdd(&tab[s].sxx[4], -0.999 * ny * nz); atomicAdd(&tab[s].sxx[5], 1.0 - 0.999 * nz * nz);
}

// AdditiveGaussianVoxel::finalize
__global__ void __launch_bounds__(256) vgicp_finalize_kernel(const NdtBuildLine* __restrict__ tab, VgLine* __restrict__ out,
                                                             unsigned long long n_lines, unsigned* __restrict__ n_vox) {
  const unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_lines) return;
  VgLine o;
  o.key = tab[s].key; o.n = 0; o.pad = 0;
  for (int k = 0; k < 3; k++) o.mean[k] = 0.0;
  for (int k = 0; k < 6; k++) o.cov[k] = 0.0;
  for (int k = 0; k < 4; k++) o.pad2[k] = 0.0;
  if (o.key != 0ull) {
    const double n = (double)tab[s].count;
    o.n = (int)tab[s].count;
    for (int k = 0; k < 3; k++) o.mean[k] = tab[s].sum[k] / n;
    for (int k = 0; k < 6; k++) o.cov[k] = tab[s].sxx[k] / n;
    atomicAdd(n_vox, 1u);
  }
  out[s] = o;
}

// One source point of a VGICP cost evaluation: update_correspondences at T with the Mahalanobis matrices stored (update)
// or reused, then linearize / compute_error (fast_vgicp_impl.hpp:72-207), double.  `corr` / `maha` point at the [n_off, n]
// correspondence slots / 6 [n_off, n] doubles of this cloud.  Shared by the single-pair kernel below (compile-time flags)
// and the batched global-alignment kernel (galign.cu, flags per candidate): the same expressions, so the same bits.
__device__ __forceinline__ void vgicp_point(const VgView& v, const float4 a, const double* __restrict__ src_nrm, int i, int n, int n_off,
                                            const Pose34d& T, int* __restrict__ corr, double* __restrict__ maha, bool update,
                                            bool deriv, double (&vals)[29]) {
  const double3 t = xform(T, a);
  int3 c = make_int3(0, 0, 0);
  double rn[3] = {0.0, 0.0, 0.0};
  if (update) {
    c = vg_coord(t.x, t.y, t.z, v.res);
    const double* na = src_nrm + 4 * (size_t)i;
    rn[0] = T.R[0] * na[0] + T.R[1] * na[1] + T.R[2] * na[2];
    rn[1] = T.R[3] * na[0] + T.R[4] * na[1] + T.R[5] * na[2];
    rn[2] = T.R[6] * na[0] + T.R[7] * na[1] + T.R[8] * na[2];
  }
#pragma unroll 1
  for (int o = 0; o < n_off; o++) {
    const size_t q = (size_t)o * n + i;
    int slot;
    if (update) {
      const int3 d = stencil_offset(o, n_off);
      slot = voxel_lookup(v, c.x + d.x, c.y + d.y, c.z + d.z);
      corr[q] = slot;
    } else {
      slot = corr[q];
    }
    if (slot < 0) continue;
    vals[28] += 1.0;
    const VgLine* ln = v.lines + slot;
    double M[3][3];
    if (update) {
      // RCR = cov_B + R cov_A R^T with cov_A = I - 0.999 n n^T
      const double A0 = ln->cov[0] + 1.0 - 0.999 * rn[0] * rn[0], A1 = ln->cov[1] - 0.999 * rn[0] * rn[1], A2 = ln->cov[2] - 0.999 * rn[0] * rn[2];
      const double A4 = ln->cov[3] + 1.0 - 0.999 * rn[1] * rn[1], A5 = ln->cov[4] - 0.999 * rn[1] * rn[2], A8 = ln->cov[5] + 1.0 - 0.999 * rn[2] * rn[2];
      const double c00 = A4 * A8 - A5 * A5, c01 = A5 * A2 - A1 * A8, c02 = A1 * A5 - A4 * A2;
      const double idet = 1.0 / (A0 * c00 + A1 * c01 + A2 * c02);
      M[0][0] = c00 * idet; M[0][1] = c01 * idet; M[0][2] = c02 * idet;
      M[1][1] = (A0 * A8 - A2 * A2) * idet; M[1][2] = (A2 * A1 - A0 * A5) * idet; M[2][2] = (A0 * A4 - A1 * A1) * idet;
      M[1][0] = M[0][1]; M[2][0] = M[0][2]; M[2][1] = M[1][2];
      double* Ms = maha + 6 * q;
      Ms[0] = M[0][0]; Ms[1] = M[0][1]; Ms[2] = M[0][2]; Ms[3] = M[1][1]; Ms[4] = M[1][2]; Ms[5] = M[2][2];
    } else {
      const double* Ms = maha + 6 * q;
      M[0][0] = Ms[0]; M[0][1] = M[1][0] = Ms[1]; M[0][2] = M[2][0] = Ms[2]; M[1][1] = Ms[3]; M[1][2] = M[2][1] = Ms[4]; M[2][2] = Ms[5];
    }
    const double w = sqrt((double)ln->n);
    accum_d2d(vals, M, make_double3(ln->mean[0] - t.x, ln->mean[1] - t.y, ln->mean[2] - t.z), t, w, deriv);
  }
}

// linearize (UPDATE: update_correspondences at T, Mahalanobis matrices stored) / compute_error (reuse).
// One thread per source point, double.
template <bool UPDATE, bool DERIV>
__global__ void __launch_bounds__(256) vgicp_cost_kernel(VgView v, const float4* __restrict__ src, const double* __restrict__ src_nrm,
                                                         int n, int n_off, Pose34d T, int* __restrict__ corr,
                                                         double* __restrict__ maha, double* __restrict__ partials,
                                                         unsigned* __restrict__ done, double* __restrict__ result, double seq,
                                                         ShardComm sc) {
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    vgicp_point(v, __ldg(src + i), src_nrm, i, n, n_off, T, corr, maha, UPDATE, DERIV, vals);
  block_partials<29>(vals, partials);
  grid_finalize<29>(partials, done, result, 0, -1, 0.0, kResSeq, seq, sc, 0);
}

// Exact nearest-neighbour distance by a scan of the whole target, for points with nothing inside the grid search radius:
// calc_fitness_score counts every point however far (max_range = DBL_MAX).  Thread version.
__device__ __forceinline__ float nn_scan_thread(const float4* __restrict__ tgt, int n_tgt, float qx, float qy, float qz) {
  float bd = 3.0e38f;
  for (int j = 0; j < n_tgt; j++) { const float4 b = __ldg(tgt + j); bd = fminf(bd, dist2(qx, qy, qz, b.x, b.y, b.z)); }
  return bd;
}
// Warp version: lanes stride over the target, then a min across lanes (every lane returns it).
__device__ __forceinline__ float nn_scan_warp(const float4* __restrict__ tgt, int n_tgt, float qx, float qy, float qz) {
  float bd = 3.0e38f;
  for (int j = threadIdx.x & 31; j < n_tgt; j += 32) { const float4 b = __ldg(tgt + j); bd = fminf(bd, dist2(qx, qy, qz, b.x, b.y, b.z)); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bd = fminf(bd, __shfl_xor_sync(0xffffffffu, bd, o));
  return bd;
}

// getFitnessScore (sum of squared 1-NN distances <= max_range, and their count) over block lb of the G blocks a cloud of n
// points gets, stored as the block's row (sum, count) of partials.  WARP: one warp per point (knn_exact_warp), else one
// thread per point (nn1_exact_thread).  tgt != nullptr: points with no neighbour within search_sq get the exact one by a
// scan of the whole target (nn_scan_*), for calc_fitness_score.  The single-pair kernel and the loop detector's batched
// kernel (loop.cu) both run this body, so a candidate's row has the single-pair bits.
template <bool WARP>
__device__ __forceinline__ void fitness_range(const MapView& mv, const float4* __restrict__ src, int n, int lb, int G, const Pose34f& Tf,
                                              float search_sq, float max_range, const float4* __restrict__ tgt, int n_tgt,
                                              double* __restrict__ partials) {
  __shared__ double s_acc[kRegWarps][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double sum = 0.0, cnt = 0.0;
  if constexpr (WARP) {
    __shared__ __align__(16) unsigned char s_list[kRegWarps * kWarpListBytes];
    WarpList wl = make_warp_list(s_list, warp);
    for (int i = lb * kRegWarps + warp; i < n; i += G * kRegWarps) {
      const float3 q = xform(Tf, __ldg(src + i));
      Neighbor nb;
      const int nf = knn_exact_warp<1>(mv, q.x, q.y, q.z, search_sq, wl, nb);
      float d2 = __shfl_sync(kFull, nb.d2, 0);
      bool found = nf > 0;
      if (!found && tgt) { d2 = nn_scan_warp(tgt, n_tgt, q.x, q.y, q.z); found = n_tgt > 0; }   // warp-uniform
      if (found && d2 <= max_range) { sum += (double)d2; cnt += 1.0; }
    }
  } else {
    for (int i = lb * blockDim.x + threadIdx.x; i < n; i += G * blockDim.x) {
      const float3 q = xform(Tf, __ldg(src + i));
      float d2; int id;
      bool found = nn1_exact_thread(mv, q.x, q.y, q.z, search_sq, &d2, &id);
      if (!found && tgt) { d2 = nn_scan_thread(tgt, n_tgt, q.x, q.y, q.z); found = n_tgt > 0; }
      if (found && d2 <= max_range) { sum += (double)d2; cnt += 1.0; }
    }
    sum = warp_sum(sum); cnt = warp_sum(cnt);
  }
  if (lane == 0) { s_acc[warp][0] = sum; s_acc[warp][1] = cnt; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double s = 0.0;
    for (int w = 0; w < kRegWarps; w++) s += s_acc[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kNV + threadIdx.x] = s;
  }
}

// getFitnessScore of one cloud: fitness_range over the whole grid, then grid_finalize.  Blocks of kRegWarps warps; the warp
// shape asks for 3 blocks per SM, the thread shape for no minimum (0).
template <bool WARP>
__global__ void __launch_bounds__(kRegWarps * 32, WARP ? 3 : 0) fitness_kernel(MapView mv, const float4* __restrict__ src, int n,
                                                                               Pose34f Tf, float search_sq, float max_range,
                                                                               double* __restrict__ partials, unsigned* __restrict__ done,
                                                                               double* __restrict__ result, double seq, ShardComm sc) {
  fitness_range<WARP>(mv, src, n, (int)blockIdx.x, (int)gridDim.x, Tf, search_sq, max_range, nullptr, 0, partials);
  grid_finalize<2>(partials, done, result, 0, -1, 0.0, kResSeq, seq, sc, 0);
}

}  // namespace lsd

// ==================================================================== host side
struct lsd_reg {
  lsd_reg_params_t p{};
  int device = 0;
  cudaStream_t stream = nullptr;
  float4 *d_src = nullptr, *d_tgt = nullptr;
  double *d_src_nrm = nullptr, *d_tgt_nrm = nullptr;  // [n,4]: smallest-eigenvalue direction of the k-NN covariance, #neighbours
  int n_src = 0, n_tgt = 0, cap_src = 0, cap_tgt = 0;
  lsd_map* tgt_map = nullptr;  // exact-NN index of the target cloud (GICP, fitness)
  lsd_map* src_map = nullptr;  // exact-NN index of the source cloud (GICP covariances)
  bool tgt_map_built = false, src_normals_built = false;
  lsd::NdtView ndt{};
  unsigned long long ndt_lines = 0;
  lsd::VgView vg{};
  unsigned long long vg_lines = 0;
  unsigned n_voxels = 0;
  int* d_corr = nullptr; size_t corr_cap = 0;
  double* d_maha = nullptr; size_t maha_cap = 0;
  double* d_partials = nullptr;
  unsigned* d_done = nullptr;
  double *h_result = nullptr, *d_result = nullptr;
  long long seq = 0;
  lsd::ShardComm sc;
  int shard_tile = 32;              // lsd_reg_shard_export: x-y tile edge in NDT voxels
  std::vector<double> iter_log;     // 4 doubles per outer LM iteration of the last align (lsd_reg_iteration_log)
  float4* d_stage = nullptr; size_t stage_cap = 0;   // staging of host clouds (lsd_reg_set_target / _source)
  int pending_world = 0;            // world announced by lsd_reg_shard_export, active after lsd_reg_shard_connect
  double* d_inbox = nullptr;        // this rank's inbox of the in-kernel all-reduce (grid_finalize)
  std::vector<void*> ipc_opened;
  double final_T[16];
  double lin_T[16];
  int converged = 0, iterations = 0;
  double final_H[36];
  long long launches = 0;
};

namespace lsd {

static void T_to_pose(const double* T, Pose34d* d, Pose34f* f) {
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) { if (d) d->R[3 * a + b] = T[4 * a + b]; if (f) f->R[3 * a + b] = (float)T[4 * a + b]; }
    if (d) d->t[a] = T[4 * a + 3];
    if (f) f->t[a] = (float)T[4 * a + 3];
  }
}

static lsd_status_t reg_wait(lsd_reg* r, double seq) { return wait_seq(r->h_result + kResSeq, r->stream, seq, 20.0); }

constexpr int kThreadShapeMin = 16384;  // clouds from this size on use the thread-per-point search kernels
static int reg_grid(int n) { return std::max(1, std::min((n + 255) / 256, kLioMaxGrid)); }
static int warp_grid(int n) { return std::max(1, std::min((n + kRegWarps - 1) / kRegWarps, lsd::kNumSms * 6)); }

// getFitnessScore's grid search radius: max_range, at most 64 map voxels
static float fitness_search_sq(double max_range, double map_resolution) {
  return (float)std::min(max_range, 64.0 * map_resolution * map_resolution * 64.0);
}

// f(std::bool_constant<update>, std::bool_constant<deriv>): launches the <UPDATE, DERIV> instance of a cost kernel
template <class F>
static void dispatch_update_deriv(bool update, bool deriv, F&& f) {
  using Y = std::true_type;
  using N = std::false_type;
  if (update && deriv) f(Y{}, Y{});
  else if (update) f(Y{}, N{});
  else if (deriv) f(N{}, Y{});
  else f(N{}, N{});
}

// H (36, symmetric) and b (6) from a cost row (upper triangle of H in 0..21, b in 21..27)
static void unpack_hb(const double* res, double* H36, double* b6) {
  int q = 0;
  for (int a = 0; a < 6; a++) for (int c = a; c < 6; c++) { H36[6 * a + c] = H36[6 * c + a] = res[q]; q++; }
  for (int a = 0; a < 6; a++) b6[a] = res[21 + a];
}

// linearize (update = true) / compute_error at T.  H36/b6 may be null.
static lsd_status_t reg_cost(lsd_reg* r, const double* T, bool update, double* H36, double* b6, double* err, int* n_corr) {
  if (r->n_src <= 0) { set_error("registration: no source cloud"); return LSD_ERR_INVALID; }
  cudaStream_t st = r->stream;
  const double seq = (double)(++r->seq);
  const bool deriv = H36 != nullptr;
  if (update) memcpy(r->lin_T, T, sizeof(r->lin_T));
  if (r->sc.world > 1 && r->p.kind != LSD_REG_NDT_P2D) { set_error("tile-sharded matching serves NDT_P2D only (GICP needs a cross-rank arg-min, not a sum)"); return LSD_ERR_INVALID; }
  if (r->p.kind == LSD_REG_NDT_P2D) {
    if (!r->ndt.lines) { set_error("registration: no target cloud"); return LSD_ERR_INVALID; }
    Pose34f lin, ev;
    T_to_pose(r->lin_T, nullptr, &lin);
    T_to_pose(T, nullptr, &ev);
    const int no = r->p.ndt_neighbors;
    const int g = reg_grid(r->n_src);
    dispatch_update_deriv(update, deriv, [&](auto U, auto D) {
      ndt_cost_kernel<decltype(U)::value, decltype(D)::value><<<g, 256, 0, st>>>(r->ndt, r->d_src, r->n_src, no, lin, ev, r->d_corr,
                                                                                 r->d_partials, r->d_done, r->d_result, seq, r->sc);
    });
    r->launches++;
  } else if (r->p.kind == LSD_REG_VGICP) {
    if (!r->vg.lines || !r->tgt_map_built) { set_error("registration: no target cloud"); return LSD_ERR_INVALID; }
    Pose34d Td;
    T_to_pose(T, &Td, nullptr);
    const int no = r->p.ndt_neighbors;
    const int g = reg_grid(r->n_src);
    dispatch_update_deriv(update, deriv, [&](auto U, auto D) {
      vgicp_cost_kernel<decltype(U)::value, decltype(D)::value><<<g, 256, 0, st>>>(r->vg, r->d_src, r->d_src_nrm, r->n_src, no, Td, r->d_corr,
                                                                                   r->d_maha, r->d_partials, r->d_done, r->d_result, seq, r->sc);
    });
    r->launches++;
  } else {
    if (!r->tgt_map_built) { set_error("registration: no target cloud"); return LSD_ERR_INVALID; }
    Pose34d Td; Pose34f Tf;
    T_to_pose(T, &Td, &Tf);
    if (update) {
      const float mc = (float)r->p.max_corr_dist;
      if (r->n_src >= kThreadShapeMin)
        gicp_corr_thread_kernel<<<(r->n_src + 255) / 256, 256, 0, st>>>(r->tgt_map->view, r->d_src, r->d_src_nrm, r->n_src, r->d_tgt_nrm, Td, Tf,
                                                                        mc * mc, r->d_corr, r->d_maha);
      else
        gicp_corr_kernel<<<warp_grid(r->n_src), kRegWarps * 32, 0, st>>>(r->tgt_map->view, r->d_src, r->d_src_nrm, r->n_src, r->d_tgt_nrm, Td, Tf,
                                                                       mc * mc, r->d_corr, r->d_maha);
      r->launches++;
    }
    const int g = reg_grid(r->n_src);
    if (deriv) gicp_cost_kernel<true><<<g, 256, 0, st>>>(r->d_src, r->n_src, r->d_tgt, Td, r->d_corr, r->d_maha, r->d_partials, r->d_done, r->d_result, seq, r->sc);
    else gicp_cost_kernel<false><<<g, 256, 0, st>>>(r->d_src, r->n_src, r->d_tgt, Td, r->d_corr, r->d_maha, r->d_partials, r->d_done, r->d_result, seq, r->sc);
    r->launches++;
  }
  LSD_CUDA(cudaGetLastError());
  lsd_status_t w = reg_wait(r, seq);
  if (w) return w;
  const double* res = r->h_result;
  if (H36) unpack_hb(res, H36, b6);
  if (err) *err = res[27];
  if (n_corr) *n_corr = (int)(res[28] + 0.5);
  return LSD_OK;
}

// ---- SE(3) helpers (double, row-major 4x4)
static void mat4_mul(const double* A, const double* B, double* C) {
  double t[16];
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) { double s = 0; for (int k = 0; k < 4; k++) s += A[4 * i + k] * B[4 * k + j]; t[4 * i + j] = s; }
  memcpy(C, t, sizeof(t));
}
// so3.hpp:60-78 + :80-104 (rotation first)
static void se3_exp(const double* a, double* T) {
  const double wx = a[0], wy = a[1], wz = a[2];
  const double theta_sq = wx * wx + wy * wy + wz * wz;
  double imag, real;
  if (theta_sq < 1e-10) {
    const double tq = theta_sq * theta_sq;
    imag = 0.5 - 1.0 / 48.0 * theta_sq + 1.0 / 3840.0 * tq;
    real = 1.0 - 1.0 / 8.0 * theta_sq + 1.0 / 384.0 * tq;
  } else {
    const double th = sqrt(theta_sq), half = 0.5 * th;
    imag = sin(half) / th; real = cos(half);
  }
  double q[4] = {imag * wx, imag * wy, imag * wz, real};
  double R[9];
  eskf::q2R(q, R);
  const double theta = sqrt(theta_sq);
  double Om[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0}, Om2[9], V[9];
  eskf::mm3(Om, Om, Om2);
  if (theta < 1e-10) {
    memcpy(V, R, sizeof(V));
  } else {
    const double c1 = (1.0 - cos(theta)) / theta_sq, c2 = (theta - sin(theta)) / (theta_sq * theta);
    for (int i = 0; i < 9; i++) V[i] = (i % 4 == 0 ? 1.0 : 0.0) + c1 * Om[i] + c2 * Om2[i];
  }
  double tv[3];
  eskf::mv3(V, a + 3, tv);
  for (int i = 0; i < 16; i++) T[i] = 0;
  for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) T[4 * i + j] = R[3 * i + j]; T[4 * i + 3] = tv[i]; }
  T[15] = 1.0;
}
// Eigen::AngleAxisd(R).angle(): via the quaternion of R
static double rot_angle(const double* T) {
  const double tr = T[0] + T[5] + T[10];
  double qw, qx, qy, qz;
  if (tr > 0) { double t = sqrt(tr + 1.0); qw = 0.5 * t; t = 0.5 / t; qx = (T[9] - T[6]) * t; qy = (T[2] - T[8]) * t; qz = (T[4] - T[1]) * t; }
  else {
    int i = 0; if (T[5] > T[0]) i = 1; if (T[10] > T[5 * i]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double t = sqrt(T[5 * i] - T[5 * j] - T[5 * k] + 1.0);
    double q[3]; q[i] = 0.5 * t; t = 0.5 / t;
    qw = (T[4 * k + j] - T[4 * j + k]) * t; q[j] = (T[4 * j + i] + T[4 * i + j]) * t; q[k] = (T[4 * k + i] + T[4 * i + k]) * t;
    qx = q[0]; qy = q[1]; qz = q[2];
  }
  const double n = sqrt(qx * qx + qy * qy + qz * qz);
  if (qw < 0) qw = -qw;  // AngleAxis(Quaternion): angle = 2 atan2(|vec|, |w|)
  return 2.0 * atan2(n, qw);
}
static bool is_converged(const lsd_reg_params_t& p, const double* delta, double scale) {  // lsq_registration_impl.hpp:112-131
  const double Rdeg = rot_angle(delta) / M_PI * 180.0;
  const double r_delta = 1.0 / (p.rotation_epsilon_deg * scale) * Rdeg;
  double t_delta = 0;
  for (int i = 0; i < 3; i++) t_delta = std::max(t_delta, fabs(delta[4 * i + 3]) / (p.transformation_epsilon * scale));
  return std::max(r_delta, t_delta) < 1;
}
// solve (H + lambda I) d = -b by LDL^T (SPD after damping)
static bool solve6(const double* H, double lambda, const double* b, double* d) {
  double A[36], L[36] = {0}, D[6];
  for (int i = 0; i < 36; i++) A[i] = H[i];
  for (int i = 0; i < 6; i++) A[7 * i] += lambda;
  for (int j = 0; j < 6; j++) {
    double s = A[7 * j];
    for (int k = 0; k < j; k++) s -= L[6 * j + k] * L[6 * j + k] * D[k];
    D[j] = s;
    if (!(fabs(s) > 0)) return false;
    L[7 * j] = 1.0;
    for (int i = j + 1; i < 6; i++) {
      double t = A[6 * i + j];
      for (int k = 0; k < j; k++) t -= L[6 * i + k] * L[6 * j + k] * D[k];
      L[6 * i + j] = t / s;
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) { double s = -b[i]; for (int k = 0; k < i; k++) s -= L[6 * i + k] * y[k]; y[i] = s; }
  for (int i = 0; i < 6; i++) y[i] /= D[i];
  for (int i = 5; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < 6; k++) s -= L[6 * k + i] * d[k]; d[i] = s; }
  return true;
}

// LsqRegistration::computeTransformation with step_lm (lsq_registration_impl.hpp:71-109,163-208) as a resumable state:
// the state names the cost evaluation it needs next (want_T, want_update: linearize with H and b, else compute_error) and
// lm_feed consumes its result.  lsd_reg_align drives one state to the end; the loop detector (loop.cu) advances a whole
// candidate set, one batched evaluation per round.  One implementation of the LM rules serves both.
struct LmState {
  lsd_reg_params_t p;
  double x0[16], lambda, nu, H[36], b[6], y0, d[6], delta[16], xi[16], final_H[36];
  int it, trial;
  bool stepped, stationary;
  int converged, iterations;
  bool done, h_set;                 // h_set: final_H holds the Hessian of an accepted step
  double want_T[16];
  bool want_update;
  std::chrono::steady_clock::time_point clock0;
  double timeout_ms;
  std::vector<double> iter_log;     // 4 doubles per outer iteration (lsd_reg_iteration_log)
};

static void lm_finish(LmState& s) { s.done = true; }

// next LM trial of the current outer iteration, or the end of the iteration when none is left
static void lm_end_outer(LmState& s);
static void lm_try_trial(LmState& s) {
  if (s.trial >= s.p.lm_max_iterations || !solve6(s.H, s.lambda, s.b, s.d)) { s.stepped = false; lm_end_outer(s); return; }
  se3_exp(s.d, s.delta);
  mat4_mul(s.delta, s.x0, s.xi);
  memcpy(s.want_T, s.xi, sizeof(s.xi));
  s.want_update = false;
}

static void lm_end_outer(LmState& s) {
  if (!s.stepped) { lm_finish(s); return; }  // "lm not converged!!"
  s.converged = is_converged(s.p, s.delta, 1.0) ? 1 : 0;
  {  // what is_converged looked at (lsd_reg_iteration_log): |t|_inf of the step, its rotation angle, the cost it started from
    double tm = 0; for (int k = 0; k < 3; k++) tm = std::max(tm, fabs(s.delta[4 * k + 3]));
    s.iter_log.push_back(tm); s.iter_log.push_back(rot_angle(s.delta) / M_PI * 180.0); s.iter_log.push_back(s.y0); s.iter_log.push_back(s.lambda);
  }
  if (s.timeout_ms > 0) {
    const double el = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - s.clock0).count();
    if (el > s.timeout_ms && is_converged(s.p, s.delta, 10.0)) { s.converged = 1; lm_finish(s); return; }
    else if (el > 1.5 * s.timeout_ms) { lm_finish(s); return; }
  }
  if (s.stationary && !s.converged) {
    // A stationary point of the reference's loop: the FIRST LM trial was rejected (rho < 0) yet small enough for
    // is_converged_low, so step_lm returned with x0 and lambda untouched (lsq_registration_impl.hpp:190-193) — and
    // the step is not small enough for is_converged.  The next iteration linearises at the same x0 with the same lambda:
    // with deterministic sums it is this iteration again, and again, to the iteration cap (measured on config 3: 60 of
    // 64 iterations, the same 1.05 cm / 0.001 deg step each; the reference's CUDA build leaves it through the run-to-run
    // noise of its fp32 atomic sums).  The outcome is known without running them: without a time budget the loop ends at
    // the cap unconverged; with one it ends when the budget is spent, converged by is_converged_low (:94-104).
    if (s.timeout_ms > 0) s.converged = 1;
    else s.iterations = s.p.max_iterations - 1;
    lm_finish(s);
    return;
  }
  s.it++;
  if (s.it >= s.p.max_iterations || s.converged) { lm_finish(s); return; }
  s.iterations = s.it;
  memcpy(s.want_T, s.x0, sizeof(s.x0));
  s.want_update = true;
}

static void lm_begin(LmState& s, const lsd_reg_params_t& p, const double* guess) {
  s.p = p;
  memcpy(s.x0, guess, sizeof(s.x0));
  s.lambda = -1.0;
  s.converged = 0;
  s.iterations = 0;
  s.it = 0;
  s.done = false;
  s.h_set = false;
  s.clock0 = std::chrono::steady_clock::now();
  s.timeout_ms = (double)(p.max_process_time_us / 1000);
  s.iter_log.clear();
  if (p.max_iterations <= 0) { lm_finish(s); return; }
  memcpy(s.want_T, s.x0, sizeof(s.x0));
  s.want_update = true;
}

// The result of the evaluation the state asked for: H/b/err of linearize(want_T), or err of compute_error(want_T).
static void lm_feed(LmState& s, const double* H, const double* b, double err) {
  if (s.want_update) {
    memcpy(s.H, H, sizeof(s.H)); memcpy(s.b, b, sizeof(s.b)); s.y0 = err;
    if (s.lambda < 0.0) { double m = 0; for (int i = 0; i < 6; i++) m = std::max(m, fabs(s.H[7 * i])); s.lambda = s.p.lm_init_lambda_factor * m; }
    s.nu = 2.0;
    s.stepped = false; s.stationary = false;
    s.trial = 0;
    lm_try_trial(s);
    return;
  }
  const double yi = err;
  double den = 0;
  for (int k = 0; k < 6; k++) den += s.d[k] * (s.lambda * s.d[k] - s.b[k]);
  const double rho = (s.y0 - yi) / den;
  if (rho < 0) {
    if (is_converged(s.p, s.delta, 10.0)) { s.stepped = true; s.stationary = (s.trial == 0); lm_end_outer(s); return; }
    s.lambda = s.nu * s.lambda; s.nu = 2 * s.nu;
    s.trial++;
    lm_try_trial(s);
    return;
  }
  memcpy(s.x0, s.xi, sizeof(s.xi));
  s.lambda = s.lambda * std::max(1.0 / 3.0, 1 - pow(2 * rho - 1, 3));
  memcpy(s.final_H, s.H, sizeof(s.H));
  s.h_set = true;
  s.stepped = true;
  lm_end_outer(s);
}

static lsd_status_t reg_align(lsd_reg* r, const double* guess) {
  LmState s;
  lm_begin(s, r->p, guess);
  r->converged = 0;
  r->iterations = 0;
  r->iter_log.clear();
  while (!s.done) {
    double H[36], b[6], y;
    lsd_status_t st = reg_cost(r, s.want_T, s.want_update, s.want_update ? H : nullptr, b, &y, nullptr);
    if (st < 0) return st;
    lm_feed(s, H, b, y);
    r->iterations = s.iterations;
  }
  r->converged = s.converged;
  r->iterations = s.iterations;
  r->iter_log.swap(s.iter_log);
  if (s.h_set) memcpy(r->final_H, s.final_H, sizeof(s.final_H));
  memcpy(r->final_T, s.x0, sizeof(s.x0));
  return LSD_OK;
}

static lsd_status_t reg_alloc_src(lsd_reg* r, int n) {
  if (n <= r->cap_src) return LSD_OK;
  cudaFree(r->d_src); cudaFree(r->d_src_nrm); cudaFree(r->d_corr); cudaFree(r->d_maha);
  r->d_src = nullptr; r->d_src_nrm = nullptr; r->d_corr = nullptr; r->d_maha = nullptr;
  const size_t c = (size_t)n + (size_t)n / 4 + 1024;
  LSD_CUDA(cudaMalloc((void**)&r->d_src, c * 16));
  LSD_CUDA(cudaMalloc((void**)&r->d_src_nrm, c * 32));
  LSD_CUDA(cudaMalloc((void**)&r->d_corr, c * 27 * sizeof(int)));
  LSD_CUDA(cudaMalloc((void**)&r->d_maha, c * 6 * sizeof(double) * (r->p.kind == LSD_REG_VGICP ? (size_t)r->p.ndt_neighbors : 1)));
  r->cap_src = (int)c;
  return LSD_OK;
}

static int auto_log2(size_t n_items, int lo, int hi) {
  int l = lo;
  while (l < hi && (1ull << l) < n_items * 2) l++;
  return l;
}

// The target's voxel map v (NdtView or VgView, v.res already set) for n points: sized from n (or map_log2_lines), its
// build table allocated and cleared, accum(build, mask, d_fail) and finalize(build, lines, d_vox) launched on the
// handle's stream.  Fails with LSD_ERR_CAPACITY when a point found no slot or lies outside the key range.
template <class View, class Accum, class Finalize>
static lsd_status_t build_voxel_table(lsd_reg* r, int n, const char* method, View& v, unsigned long long& n_lines, Accum accum,
                                      Finalize finalize) {
  cudaStream_t st = r->stream;
  const int l2 = r->p.map_log2_lines > 0 ? r->p.map_log2_lines : auto_log2((size_t)n / 2 + 1024, 12, 27);
  const unsigned long long lines = 1ull << l2;
  NdtBuildLine* build = nullptr;
  LSD_CUDA(cudaMalloc((void**)&build, lines * sizeof(NdtBuildLine)));
  LSD_CUDA(cudaMemsetAsync(build, 0, lines * sizeof(NdtBuildLine), st));
  if (n_lines != lines) {
    cudaFree(v.lines); v.lines = nullptr;
    LSD_CUDA(cudaMalloc((void**)&v.lines, lines * sizeof(*v.lines)));
    n_lines = lines;
  }
  v.mask = lines - 1;
  unsigned* d_cnt = reinterpret_cast<unsigned*>(r->d_done) + 4;
  LSD_CUDA(cudaMemsetAsync(d_cnt, 0, 8, st));
  accum(build, lines - 1, d_cnt);
  finalize(build, lines, d_cnt + 1);
  r->launches += 2;
  unsigned h[2] = {0, 0};
  LSD_CUDA(cudaMemcpyAsync(h, d_cnt, 8, cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  LSD_CUDA(cudaFree(build));
  r->n_voxels = h[1];
  if (h[0]) { set_error("%s voxel table too small / coordinates out of range: %u points dropped (raise map_log2_lines)", method, h[0]); return LSD_ERR_CAPACITY; }
  return LSD_OK;
}

}  // namespace lsd

using namespace lsd;

extern "C" {

void lsd_reg_default_params(lsd_reg_params_t* p, int kind) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->kind = kind;
  p->max_iterations = 64;                 // registrations.cpp:39,111
  p->transformation_epsilon = 0.01;       // registrations.cpp:38,109
  p->lm_max_iterations = 10;              // lsq_registration.hpp (lm_max_iterations_)
  p->lm_init_lambda_factor = 1e-9;        // lsq_registration.hpp (lm_init_lambda_factor_)
  p->max_process_time_us = 0;
  p->k_correspondences = 20;              // registrations.cpp:41
  p->max_corr_dist = 2.0;                 // registrations.cpp:40 (0.5 in loop closure, loop_detector.hpp:59)
  p->normal_search_sq = 25.0;
  p->map_resolution = 0.5;
  p->map_log2_lines = 0;                  // auto
  if (kind == LSD_REG_NDT_P2D) {
    p->rotation_epsilon_deg = 0.1;        // registrations.cpp:110
    p->resolution = 1.0;                  // registrations.cpp:106
    p->ndt_neighbors = 7;                 // DIRECT7, registrations.cpp:114
  } else if (kind == LSD_REG_VGICP) {
    p->transformation_epsilon = 0.1;      // registrations.cpp:61
    p->rotation_epsilon_deg = 0.1;        // registrations.cpp:62
    p->resolution = 1.0;                  // registrations.cpp:60
    p->ndt_neighbors = 1;                 // DIRECT1, fast_vgicp_impl.hpp:23
  } else {
    p->rotation_epsilon_deg = 1e-2;       // LsqRegistration default (lsq_registration_impl.hpp:24), compared against degrees (:113-116)
    p->resolution = 1.0;
    p->ndt_neighbors = 1;
  }
}

lsd_status_t lsd_reg_create(lsd_reg_t** out, const lsd_reg_params_t* p) {
  if (!out || !p || (p->kind != LSD_REG_NDT_P2D && p->kind != LSD_REG_GICP && p->kind != LSD_REG_VGICP) || p->resolution <= 0 ||
      (p->ndt_neighbors != 1 && p->ndt_neighbors != 7 && p->ndt_neighbors != 27) || p->k_correspondences < 3 || p->k_correspondences > 20) {
    set_error("lsd_reg_create: bad params (kind, resolution, ndt_neighbors in {1,7,27}, 3 <= k <= 20)");
    return LSD_ERR_INVALID;
  }
  lsd_status_t s = ensure_device();
  if (s) return s;
  s = upload_stencils();
  if (s) return s;
  lsd_reg* r = new lsd_reg();
  r->p = *p;
  cudaGetDevice(&r->device);
  memset(&r->sc, 0, sizeof(r->sc));
  r->sc.world = 1;
  for (int i = 0; i < 16; i++) r->final_T[i] = r->lin_T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  cudaError_t e = cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc((void**)&r->d_partials, (size_t)(lsd::kNumSms * 6 + 8) * kNV * 8);
  if (e == cudaSuccess) e = cudaMalloc((void**)&r->d_done, 64);
  if (e == cudaSuccess) e = cudaMemset(r->d_done, 0, 64);
  if (e == cudaSuccess) e = cudaHostAlloc((void**)&r->h_result, kResDoubles * 8, cudaHostAllocMapped);
  if (e == cudaSuccess) { memset(r->h_result, 0, kResDoubles * 8); e = cudaHostGetDevicePointer((void**)&r->d_result, r->h_result, 0); }
  if (e != cudaSuccess) { lsd_status_t rr = cuda_fail(e, "lsd_reg_create", __FILE__, __LINE__); lsd_reg_destroy(r); return rr; }
  *out = r;
  return LSD_OK;
}

lsd_status_t lsd_reg_destroy(lsd_reg_t* r) {
  if (!r) return LSD_OK;
  cudaSetDevice(r->device);
  if (r->stream) cudaStreamSynchronize(r->stream);
  void* ptrs[] = {r->d_src, r->d_tgt, r->d_src_nrm, r->d_tgt_nrm, r->ndt.lines, r->vg.lines, r->d_corr, r->d_maha, r->d_partials, r->d_done};
  for (void* p : ptrs) cudaFree(p);
  cudaFreeHost(r->h_result);
  for (void* q : r->ipc_opened) cudaIpcCloseMemHandle(q);
  cudaFree(r->d_inbox); cudaFree(r->d_stage);
  if (r->tgt_map) lsd_map_destroy(r->tgt_map);
  if (r->src_map) lsd_map_destroy(r->src_map);
  if (r->stream) cudaStreamDestroy(r->stream);
  delete r;
  return LSD_OK;
}

// Tile-sharded NDT target (SURVEY.md section 8e row C3; include/lsdreg.h "Tile-sharded matcher").  Same hand-shake as
// lsd_lio_shard_*: export a blob naming this rank's inbox, all-gather, connect.  Same-process peers use raw pointers.
struct RegShardBlob { long long pid; unsigned long long inbox; cudaIpcMemHandle_t h_inbox; };
static_assert(sizeof(RegShardBlob) <= LSD_SHARD_BLOB_BYTES, "LSD_SHARD_BLOB_BYTES too small");

lsd_status_t lsd_reg_shard_export(lsd_reg_t* r, int rank, int world, int tile_cells, unsigned char* blob_out) {
  if (!r || !blob_out || world < 1 || world > kMaxRanks || rank < 0 || rank >= world || tile_cells < 1) { set_error("lsd_reg_shard_export: bad rank / world (max %d ranks) / tile", kMaxRanks); return LSD_ERR_INVALID; }
  if (r->p.kind != LSD_REG_NDT_P2D) { set_error("lsd_reg_shard_export: tile sharding serves NDT_P2D only"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(r->device));
  if (!r->d_inbox) {
    LSD_CUDA(cudaMalloc((void**)&r->d_inbox, 2 * kInboxRegion * sizeof(double)));
    LSD_CUDA(cudaMemset(r->d_inbox, 0, 2 * kInboxRegion * sizeof(double)));
    LSD_CUDA(cudaDeviceSynchronize());
  }
  RegShardBlob b;
  memset(&b, 0, sizeof(b));
  b.pid = (long long)getpid();
  b.inbox = (unsigned long long)r->d_inbox;
  LSD_CUDA(cudaIpcGetMemHandle(&b.h_inbox, r->d_inbox));
  memset(blob_out, 0, LSD_SHARD_BLOB_BYTES);
  memcpy(blob_out, &b, sizeof(b));
  memset(&r->sc, 0, sizeof(r->sc));
  r->sc.rank = rank; r->sc.world = 1;      // not connected yet: lsd_reg_shard_connect sets the world
  r->shard_tile = tile_cells;
  r->pending_world = world;
  return LSD_OK;
}

lsd_status_t lsd_reg_shard_connect(lsd_reg_t* r, const unsigned char* blobs) {
  if (!r || !blobs || r->pending_world < 1 || !r->d_inbox) { set_error("lsd_reg_shard_connect: call lsd_reg_shard_export first"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(r->device));
  ShardComm sc;
  memset(&sc, 0, sizeof(sc));
  sc.rank = r->sc.rank; sc.world = r->pending_world;
  for (int p = 0; p < sc.world; p++) {
    RegShardBlob b;
    memcpy(&b, blobs + (size_t)p * LSD_SHARD_BLOB_BYTES, sizeof(b));
    if (p == sc.rank) { sc.inbox[p] = r->d_inbox; continue; }
    if (b.pid == (long long)getpid()) {
      sc.inbox[p] = reinterpret_cast<double*>(b.inbox);
      cudaPointerAttributes at;
      if (cudaPointerGetAttributes(&at, sc.inbox[p]) == cudaSuccess && at.device != r->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return cuda_fail(e, "cudaDeviceEnablePeerAccess", __FILE__, __LINE__);
        cudaGetLastError();
      }
    } else {
      void* pi = nullptr;
      LSD_CUDA(cudaIpcOpenMemHandle(&pi, b.h_inbox, cudaIpcMemLazyEnablePeerAccess));
      sc.inbox[p] = static_cast<double*>(pi);
      r->ipc_opened.push_back(pi);
    }
  }
  r->sc = sc;
  r->seq = 0;                       // all ranks restart their sequence numbers together
  r->h_result[kResSeq] = 0.0;
  return LSD_OK;
}

static lsd_status_t build_point_map(lsd_reg* r, lsd_map** mp, const float4* d_pts, int n) {
  const int l2 = r->p.map_log2_lines > 0 ? r->p.map_log2_lines : auto_log2((size_t)n, 12, 26);
  if (*mp && (*mp)->n_lines == (1ull << l2)) {
    // same table size as the previous cloud (a batch of equally sized submaps, config 4): reset in place on the handle's
    // stream — two memsets instead of cudaFree + cudaMalloc + a synchronising clear per call
    lsd_map* m = *mp;
    LSD_CUDA(cudaMemsetAsync(m->view.lines, 0, m->n_lines * sizeof(CellLine), r->stream));
    LSD_CUDA(cudaMemsetAsync(m->view.tags, 0, m->n_lines, r->stream));
    LSD_CUDA(cudaMemsetAsync(m->view.counters, 0, 4 * sizeof(unsigned long long), r->stream));
  } else {
    if (*mp) { lsd_map_destroy(*mp); *mp = nullptr; }
    lsd_status_t s = lsd_map_create(mp, (float)r->p.map_resolution, l2);
    if (s) return s;
    cudaStreamDestroy((*mp)->stream);
    (*mp)->stream = nullptr;
  }
  lsd_status_t s = launch_insert(*mp, d_pts, n, 0, r->stream);
  (*mp)->stream = nullptr;
  return s;
}

static void detach_map_stream(lsd_map* m) { if (m) m->stream = nullptr; }

// calculate_covariances (fast_gicp_impl.hpp:244-303) of the cloud d_pts: its exact-NN point map built into *mp, then the
// k-NN covariance of every point as its smallest-eigenvalue direction and neighbour count in nrm [n, 4], on the handle's
// stream.  GICP / VGICP sources and targets of lsd_reg, and the key frames of the global aligner (galign.cu).
static lsd_status_t gicp_covariances(lsd_reg* r, lsd_map** mp, const float4* d_pts, int n, double* nrm) {
  lsd_status_t s = build_point_map(r, mp, d_pts, n);
  if (s) return s;
  cudaStream_t st = r->stream;
  gicp_normals_kernel<<<warp_grid(n), kRegWarps * 32, 0, st>>>((*mp)->view, d_pts, n, r->p.k_correspondences, (float)r->p.normal_search_sq, nrm);
  gicp_normals_complete_kernel<<<warp_grid(n), kRegWarps * 32, 0, st>>>(d_pts, n, r->p.k_correspondences, nrm);
  LSD_CUDA(cudaGetLastError());
  r->launches += 3;
  return LSD_OK;
}

// GaussianVoxelMap::create_voxelmap (built lazily by the reference, fast_vgicp_impl.hpp:121-124) of the target d_pts with
// its covariances nrm into vg (lines reallocated when the size changes), at the handle's resolution.
static lsd_status_t vgicp_voxel_table(lsd_reg* r, const float4* d_pts, const double* nrm, int n, VgView& vg, unsigned long long& vg_lines) {
  cudaStream_t st = r->stream;
  vg.res = r->p.resolution;
  return build_voxel_table(r, n, "VGICP", vg, vg_lines,
      [&](NdtBuildLine* build, unsigned long long mask, unsigned* d_fail) {
        vgicp_accum_kernel<<<(n + 255) / 256, 256, 0, st>>>(build, mask, vg.res, d_pts, nrm, n, d_fail);
      },
      [&](const NdtBuildLine* build, unsigned long long lines, unsigned* d_vox) {
        vgicp_finalize_kernel<<<(unsigned)((lines + 255) / 256), 256, 0, st>>>(build, vg.lines, lines, d_vox);
      });
}

// setInputTarget: NDT builds the Gaussian voxel map immediately (ndt_cuda.cu:105-114); GICP indexes the
// cloud and computes its covariances (fast_gicp_impl.hpp:112-114).
lsd_status_t lsd_reg_set_target_dev(lsd_reg_t* r, const float* pts_dev, int n) {
  if (!r || n <= 0 || !pts_dev) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = r->stream;
  if (n > r->cap_tgt) {
    cudaFree(r->d_tgt); cudaFree(r->d_tgt_nrm); r->d_tgt = nullptr; r->d_tgt_nrm = nullptr;
    LSD_CUDA(cudaMalloc((void**)&r->d_tgt, (size_t)n * 16));
    LSD_CUDA(cudaMalloc((void**)&r->d_tgt_nrm, (size_t)n * 32));
    r->cap_tgt = n;
  }
  LSD_CUDA(cudaMemcpyAsync(r->d_tgt, pts_dev, (size_t)n * 16, cudaMemcpyDeviceToDevice, st));
  r->n_tgt = n;
  r->tgt_map_built = false;
  if (r->p.kind == LSD_REG_NDT_P2D) {
    r->ndt.res = (float)r->p.resolution;
    lsd_status_t s = build_voxel_table(r, n, "NDT", r->ndt, r->ndt_lines,
        [&](NdtBuildLine* build, unsigned long long mask, unsigned* d_fail) {
          ndt_accum_kernel<<<(n + 255) / 256, 256, 0, st>>>(build, mask, r->ndt.res, r->d_tgt, n, d_fail, r->sc.rank, r->sc.world, r->shard_tile);
        },
        [&](const NdtBuildLine* build, unsigned long long lines, unsigned* d_vox) {
          ndt_finalize_kernel<<<(unsigned)((lines + 255) / 256), 256, 0, st>>>(build, r->ndt.lines, lines, d_vox);
        });
    if (s) return s;
  } else {
    lsd_status_t s = gicp_covariances(r, &r->tgt_map, r->d_tgt, n, r->d_tgt_nrm);
    if (s) return s;
    r->tgt_map_built = true;
    if (r->p.kind == LSD_REG_VGICP) {
      s = vgicp_voxel_table(r, r->d_tgt, r->d_tgt_nrm, n, r->vg, r->vg_lines);
      if (s) return s;
    }
    LSD_CUDA(cudaStreamSynchronize(st));
  }
  return LSD_OK;
}

lsd_status_t lsd_reg_set_source_dev(lsd_reg_t* r, const float* pts_dev, int n) {
  if (!r || n <= 0 || !pts_dev) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  lsd_status_t s = reg_alloc_src(r, n);
  if (s) return s;
  cudaStream_t st = r->stream;
  LSD_CUDA(cudaMemcpyAsync(r->d_src, pts_dev, (size_t)n * 16, cudaMemcpyDeviceToDevice, st));
  r->n_src = n;
  if (r->p.kind != LSD_REG_NDT_P2D) {  // source covariances (fast_gicp_impl.hpp:109-111)
    s = gicp_covariances(r, &r->src_map, r->d_src, n, r->d_src_nrm);
    if (s) return s;
    LSD_CUDA(cudaStreamSynchronize(st));
  }
  return LSD_OK;
}

// host-pointer entry points: a staging buffer that lives with the handle (grown on demand, never shrunk)
static lsd_status_t stage_host(lsd_reg* r, const float* host, int n, float4** tmp) {
  if ((size_t)n > r->stage_cap) {
    cudaFree(r->d_stage); r->d_stage = nullptr; r->stage_cap = 0;
    LSD_CUDA(cudaMalloc((void**)&r->d_stage, (size_t)n * 16));
    r->stage_cap = (size_t)n;
  }
  *tmp = r->d_stage;
  LSD_CUDA(cudaMemcpyAsync(*tmp, host, (size_t)n * 16, cudaMemcpyHostToDevice, r->stream));
  return LSD_OK;
}
lsd_status_t lsd_reg_set_target(lsd_reg_t* r, const float* pts_host, int n) {
  if (!r || n <= 0 || !pts_host) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  float4* tmp = nullptr;
  lsd_status_t s = stage_host(r, pts_host, n, &tmp);
  if (!s) s = lsd_reg_set_target_dev(r, reinterpret_cast<const float*>(tmp), n);
  cudaStreamSynchronize(r->stream);
  return s;
}
lsd_status_t lsd_reg_set_source(lsd_reg_t* r, const float* pts_host, int n) {
  if (!r || n <= 0 || !pts_host) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  float4* tmp = nullptr;
  lsd_status_t s = stage_host(r, pts_host, n, &tmp);
  if (!s) s = lsd_reg_set_source_dev(r, reinterpret_cast<const float*>(tmp), n);
  cudaStreamSynchronize(r->stream);
  return s;
}

lsd_status_t lsd_reg_set_max_correspondence_distance(lsd_reg_t* r, double d) { if (!r || d <= 0) return LSD_ERR_INVALID; r->p.max_corr_dist = d; return LSD_OK; }

lsd_status_t lsd_reg_cost(lsd_reg_t* r, const double* T16, int update, double* H36, double* b6, double* err, int* n_corr) {
  if (!r || !T16) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  return reg_cost(r, T16, update != 0, H36, H36 ? b6 : nullptr, err, n_corr);
}

lsd_status_t lsd_reg_align(lsd_reg_t* r, const float* guess16, float* out16, int* converged, int* iterations) {
  if (!r || !guess16 || !out16) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  double g[16];
  for (int i = 0; i < 16; i++) g[i] = (double)guess16[i];
  lsd_status_t s = reg_align(r, g);
  if (s < 0) return s;
  for (int i = 0; i < 16; i++) out16[i] = (float)r->final_T[i];
  if (converged) *converged = r->converged;
  if (iterations) *iterations = r->iterations;
  return LSD_OK;
}

lsd_status_t lsd_reg_iteration_log(lsd_reg_t* r, double* out4_per_iter, int cap_iters, int* n_iters) {
  if (!r || !n_iters) return LSD_ERR_INVALID;
  const int n = (int)(r->iter_log.size() / 4);
  *n_iters = n;
  if (out4_per_iter) memcpy(out4_per_iter, r->iter_log.data(), (size_t)std::min(n, std::max(cap_iters, 0)) * 4 * sizeof(double));
  return LSD_OK;
}
lsd_status_t lsd_reg_get_final(lsd_reg_t* r, double* T16, double* H36) {
  if (!r) return LSD_ERR_INVALID;
  if (T16) memcpy(T16, r->final_T, sizeof(r->final_T));
  if (H36) memcpy(H36, r->final_H, sizeof(r->final_H));
  return LSD_OK;
}

lsd_status_t lsd_reg_fitness(lsd_reg_t* r, const double* T16_or_null, double max_range, double* score) {
  if (!r || !score || r->n_src <= 0 || r->n_tgt <= 0) return LSD_ERR_INVALID;
  if (r->sc.world > 1) { set_error("lsd_reg_fitness: not available on a tile-sharded handle (a nearest neighbour is an arg-min across ranks, not a sum)"); return LSD_ERR_INVALID; }
  LSD_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = r->stream;
  if (!r->tgt_map_built) {
    lsd_status_t s = build_point_map(r, &r->tgt_map, r->d_tgt, r->n_tgt);
    if (s) return s;
    r->launches++;
    r->tgt_map_built = true;
  }
  Pose34f Tf;
  T_to_pose(T16_or_null ? T16_or_null : r->final_T, nullptr, &Tf);
  const double seq = (double)(++r->seq);
  const float search_sq = fitness_search_sq(max_range, r->p.map_resolution);
  if (r->n_src >= kThreadShapeMin)
    fitness_kernel<false><<<reg_grid(r->n_src), kRegWarps * 32, 0, st>>>(r->tgt_map->view, r->d_src, r->n_src, Tf, search_sq, (float)max_range,
                                                                         r->d_partials, r->d_done, r->d_result, seq, r->sc);
  else
    fitness_kernel<true><<<warp_grid(r->n_src), kRegWarps * 32, 0, st>>>(r->tgt_map->view, r->d_src, r->n_src, Tf, search_sq, (float)max_range,
                                                                        r->d_partials, r->d_done, r->d_result, seq, r->sc);
  LSD_CUDA(cudaGetLastError());
  r->launches++;
  lsd_status_t w = reg_wait(r, seq);
  if (w) return w;
  const double sum = r->h_result[0], cnt = r->h_result[1];
  *score = cnt > 0 ? sum / cnt : DBL_MAX;
  return LSD_OK;
}

lsd_status_t lsd_reg_get_correspondences(lsd_reg_t* r, int32_t* corr_host, int cap, int* n) {
  if (!r || !n || (cap > 0 && !corr_host)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(r->device));
  const int per = r->p.kind == LSD_REG_GICP ? 1 : r->p.ndt_neighbors;
  *n = r->n_src * per;
  const int c = std::min(cap, *n);
  if (c > 0) LSD_CUDA(cudaMemcpyAsync(corr_host, r->d_corr, (size_t)c * 4, cudaMemcpyDeviceToHost, r->stream));
  LSD_CUDA(cudaStreamSynchronize(r->stream));
  return LSD_OK;
}

lsd_status_t lsd_reg_stats(lsd_reg_t* r, int* n_voxels, long long* launches) {
  if (!r) return LSD_ERR_INVALID;
  if (n_voxels) *n_voxels = (int)r->n_voxels;
  if (launches) *launches = r->launches;
  return LSD_OK;
}

}  // extern "C"
