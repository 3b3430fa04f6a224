// floor.cu — floor detection: prefilter, height clip, k = 10 normal filter and RANSAC plane fit, one frame per call.
//
// Replaces (PCL 1.9.1 semantics, restated in DESIGN.md section 5f; PCL is not vendored in the reference tree):
//   FloorDetectionNodelet::detect (slam/backend/hdl_graph_slam/apps/floor_detection_nodelet.cpp:79-193), the "FLIO Floor"
//     thread's per-frame work (slam/mapping/fastlio/src/fastlio.cpp:279-292) after PrefilteringNodelet (prefiltering_nodelet.cpp:
//     91-165: VoxelGrid at `resolution`, then 0.1 < |p| < 100);
//   detect_ground (slam/src/graph_utils.cpp:299-382) and its copy in MapRender (localization/map_render/map_render.cpp:81-134,
//     RANSAC threshold 0.2), which also return the inlier cloud.
//
// Pipeline, on the handle's stream:
//   [voxel grid (voxelgrid.cu)] -> floor_clip_kernel: distance filter + the two PlaneClipper3D passes, order-preserving
//   compaction of both outputs in one chained kernel, the clipped points inserted into the handle's hash-voxel map as they
//   are placed -> floor_normals_kernel: exact 10-NN on the map (knn_exact_warp<10>), the fp32 one-pass covariance in neighbour
//   order, pcl::eigen33, the viewpoint flip and the |n_z| test -> floor_complete_kernel: the exact whole-cloud 10-NN for the
//   points the grid search did not serve (all of them when the map dropped points, DESIGN.md section 5e) -> floor_compact_kernel
//   (candidates) -> per batch of B hypotheses: floor_sample_kernel (one warp: boost::mt19937 + drawIndexSample + isSampleGood +
//   computeModelCoefficients) and floor_score_kernel (every hypothesis against every candidate, counts to mapped rows) -> the
//   host replays RandomSampleConsensus::computeModel's stop rule on the counts -> floor_compact_kernel (inliers of the best).
#include <cmath>
#include <climits>
#include <vector>

#include "knn.cuh"
#include "map.h"
#include "voxelgrid.h"

namespace lsd {

constexpr int kFloorBlock = 256;
constexpr int kFloorWarps = 8;
constexpr int kFloorK = 10;              // NormalEstimation::setKSearch(10)
constexpr float kFloorMapRes = 0.5f;     // voxel of the normals' point map
constexpr float kFloorSearchSq = 4.0f;   // grid search radius^2; points with fewer than 10 inside are completed exactly
constexpr int kMtN = 624;
constexpr int kMaxHypBatch = 12288;      // the scoring kernel's per-hypothesis counts fill at most 48 KB of shared memory

struct FloorHyp { int idx[3]; int flag; float c[4]; };      // flag: 1 model, 0 skipped (collinear), -1 no sample could be drawn
struct FloorRow { int count; int flag; float c[4]; };        // mapped result row of one scored hypothesis
struct FloorRng { unsigned mt[kMtN]; int pos; int done; int s[3]; };

// ------------------------------------------------------------------ compaction chain (as keyframe_filter_kernel)
// Blocks take a ticket; block t waits for block t-1's published running totals.  Two outputs per point (a ⊇ b), their
// totals packed in one 64-bit prefix word: bit 63 published, bits 32..62 total a, bits 0..31 total b.
struct ChainOut { unsigned a, b; };
__device__ __forceinline__ ChainOut chain_place(bool ka, bool kb, unsigned b_idx, int last, unsigned long long* prefix,
                                                int* n_a, int* n_b, unsigned* s_wa, unsigned* s_wb, unsigned* s_base) {
  const unsigned ba = __ballot_sync(kFull, ka), bb = __ballot_sync(kFull, kb);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_wa[warp] = __popc(ba); s_wb[warp] = __popc(bb); }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned ta = 0, tb = 0;
    for (int w = 0; w < kFloorBlock / 32; w++) {
      const unsigned ca = s_wa[w], cb = s_wb[w];
      s_wa[w] = ta; s_wb[w] = tb; ta += ca; tb += cb;
    }
    unsigned long long base = 0ull;
    if (b_idx > 0) {
      volatile unsigned long long* pp = prefix + (b_idx - 1);
      unsigned long long v;
      while (((v = *pp) >> 63) == 0ull) {}
      base = v & 0x7fffffffffffffffull;
    }
    const unsigned long long incl = base + ((unsigned long long)ta << 32) + tb;
    __threadfence();
    prefix[b_idx] = incl | (1ull << 63);
    s_base[0] = (unsigned)(base >> 32); s_base[1] = (unsigned)(base & 0xffffffffull);
    if (last) { if (n_a) *n_a = (int)(incl >> 32); *n_b = (int)(incl & 0xffffffffull); }
  }
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
  return ChainOut{s_base[0] + s_wa[warp] + __popc(ba & lt), s_base[1] + s_wb[warp] + __popc(bb & lt)};
}

// The prefiltered cloud (distance filter on the voxel grid's output, when enabled) and the height clip; the clipped points are
// inserted into the map with id = their clipped index.  n = *n_dev when n_dev is given (the voxel grid's count), else n_host.
__global__ void __launch_bounds__(kFloorBlock) floor_clip_kernel(const float4* __restrict__ in, const int* __restrict__ n_dev, int n_host,
                                                                 int use_dist, double near_d, double far_d, float keep_d, float cut_d,
                                                                 float4* __restrict__ out_pre, float4* __restrict__ out_clip, MapView mv,
                                                                 unsigned* __restrict__ ticket, unsigned long long* __restrict__ prefix,
                                                                 int* __restrict__ n_pre, int* __restrict__ n_clip) {
  __shared__ unsigned s_ticket, s_wa[kFloorBlock / 32], s_wb[kFloorBlock / 32], s_base[2];
  if (threadIdx.x == 0) s_ticket = atomicAdd(ticket, 1u);
  __syncthreads();
  const unsigned b = s_ticket;
  const int n = n_dev ? *n_dev : n_host;
  const int i = (int)(b * kFloorBlock + threadIdx.x);
  bool ka = false, kb = false;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n) {
    p = __ldg(in + i);
    ka = true;
    if (use_dist) {
      // PrefilteringNodelet::distance_filter: double d = p.getVector3fMap().norm()
      const double d = (double)sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)), __fmul_rn(p.z, p.z)));
      ka = d > near_d && d < far_d;
    }
    // PlaneClipper3D::clipPoint3D: n . p >= -d with n = (0, 0, 1), in float; the second plane's points are removed
    const float h = __fadd_rn(__fadd_rn(__fmul_rn(0.f, p.x), __fmul_rn(0.f, p.y)), __fmul_rn(1.f, p.z));
    kb = ka && h >= -keep_d && !(h >= -cut_d);
  }
  const ChainOut o = chain_place(ka, kb, b, b == gridDim.x - 1, prefix, n_pre, n_clip, s_wa, s_wb, s_base);
  if (ka && out_pre) out_pre[o.a] = p;
  if (kb) {
    out_clip[o.b] = p;
    map_insert_point(mv, p.x, p.y, p.z, (int)o.b);
  }
}

// Order-preserving compaction of the first *n_dev points: by flag (keep != nullptr), the inliers of plane model->c
// (selectWithinDistance: double(fabsf(dot4(c, (x, y, z, 1)))) < threshold), or all of them (neither given).  ids_out
// (optional) receives 0, 1, 2, ...: the initial shuffled_indices_ of the sampler.
__device__ __forceinline__ float plane_dist(const float* c, float4 p) {
  // Eigen's SSE 4-dot: (a0 + a2) + (a1 + a3), a3 = c3 * 1
  return __fadd_rn(__fadd_rn(__fmul_rn(c[0], p.x), __fmul_rn(c[2], p.z)), __fadd_rn(__fmul_rn(c[1], p.y), __fmul_rn(c[3], 1.0f)));
}
__global__ void __launch_bounds__(kFloorBlock) floor_compact_kernel(const float4* __restrict__ in, const int* __restrict__ n_dev,
                                                                    const unsigned char* __restrict__ keep, const FloorHyp* __restrict__ model,
                                                                    double threshold, float4* __restrict__ out, int* __restrict__ ids_out,
                                                                    unsigned* __restrict__ ticket, unsigned long long* __restrict__ prefix,
                                                                    int* __restrict__ n_out) {
  __shared__ unsigned s_ticket, s_wa[kFloorBlock / 32], s_wb[kFloorBlock / 32], s_base[2];
  if (threadIdx.x == 0) s_ticket = atomicAdd(ticket, 1u);
  __syncthreads();
  const unsigned b = s_ticket;
  const int n = *n_dev;
  const int i = (int)(b * kFloorBlock + threadIdx.x);
  bool k = false;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n) {
    p = __ldg(in + i);
    if (keep) k = keep[i] != 0;
    else if (model) { const float c[4] = {model->c[0], model->c[1], model->c[2], model->c[3]}; k = (double)fabsf(plane_dist(c, p)) < threshold; }
    else k = true;
  }
  const ChainOut o = chain_place(k, k, b, b == gridDim.x - 1, prefix, nullptr, n_out, s_wa, s_wb, s_base);
  if (k) { out[o.b] = p; if (ids_out) ids_out[o.b] = (int)o.b; }
}

// ------------------------------------------------------------------ normals (NormalEstimation, k = 10)
// pcl::computeRoots2 / computeRoots / eigen33 (common/impl/eigen.hpp) in float, literally.
__device__ __forceinline__ void roots2(float b, float c, float r[3]) {
  r[0] = 0.f;
  float d = (float)((double)__fmul_rn(b, b) - 4.0 * (double)c);
  if (d < 0.f) d = 0.f;
  const float sd = sqrtf(d);
  r[2] = __fmul_rn(0.5f, __fadd_rn(b, sd));
  r[1] = __fmul_rn(0.5f, __fsub_rn(b, sd));
}
__device__ __forceinline__ void compute_roots(const float m[9], float r[3]) {
  const float m00 = m[0], m01 = m[1], m02 = m[2], m11 = m[4], m12 = m[5], m22 = m[8];
  const float c0 = m00 * m11 * m22 + 2.f * m01 * m02 * m12 - m00 * m12 * m12 - m11 * m02 * m02 - m22 * m01 * m01;
  const float c1 = m00 * m11 - m01 * m01 + m00 * m22 - m02 * m02 + m11 * m22 - m12 * m12;
  const float c2 = m00 + m11 + m22;
  if (fabsf(c0) < 1.1920928955078125e-07f) { roots2(c2, c1, r); return; }
  const float s_inv3 = (float)(1.0 / 3.0), s_sqrt3 = sqrtf(3.0f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.f) a_over_3 = 0.f;
  const float half_b = 0.5f * (c0 + c2_over_3 * (2.f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.f) q = 0.f;
  const float rho = sqrtf(-a_over_3);
  const float theta = atan2f(sqrtf(-q), half_b) * s_inv3;
  // std::cos / std::sin of a float in [0, pi/3], evaluated in double and rounded: within an ulp of the host's libm.  (sinf and
  // cosf would link a range-reduction table of their own, which moves the constant-bank slots of every kernel using sin/cos.)
  const float ct = (float)cos((double)theta), st = (float)sin((double)theta);
  r[0] = c2_over_3 + 2.f * rho * ct;
  r[1] = c2_over_3 - rho * (ct + s_sqrt3 * st);
  r[2] = c2_over_3 - rho * (ct - s_sqrt3 * st);
  float t;
  if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  if (r[1] >= r[2]) {
    t = r[1]; r[1] = r[2]; r[2] = t;
    if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  }
  if (r[0] <= 0.f) roots2(c2, c1, r);
}
__device__ __forceinline__ void eigen33_smallest(const float C[9], float& lambda, float v[3]) {
  float scale = 0.f;
  for (int j = 0; j < 9; j++) scale = fmaxf(scale, fabsf(C[j]));
  if (scale <= 1.17549435e-38f) scale = 1.f;
  float S[9];
  for (int j = 0; j < 9; j++) S[j] = C[j] / scale;
  float r[3];
  compute_roots(S, r);
  lambda = r[0] * scale;
  S[0] -= r[0]; S[4] -= r[0]; S[8] -= r[0];
  auto cross = [](const float* a, const float* b, float* o) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
  };
  float v1[3], v2[3], v3[3];
  cross(S, S + 3, v1); cross(S, S + 6, v2); cross(S + 3, S + 6, v3);
  const float l1 = v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2];
  const float l2 = v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2];
  const float l3 = v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2];
  const float* w; float l;
  if (l1 >= l2 && l1 >= l3) { w = v1; l = l1; }
  else if (l2 >= l1 && l2 >= l3) { w = v2; l = l2; }
  else { w = v3; l = l3; }
  const float s = sqrtf(l);
  v[0] = w[0] / s; v[1] = w[1] / s; v[2] = w[2] / s;
}

// Lanes 0 .. nf-1 hold the neighbours of clipped point i in (d2, index) order.  computeMeanAndCovarianceMatrix (fp32, one pass,
// neighbour order), solvePlaneParameters, flipNormalTowardsViewpoint, and normal_filtering's test; lane 0 stores.
__device__ __forceinline__ void floor_point_normal(float x, float y, float z, int nf, int i, float4 p, float vpz, double cos_thr,
                                                   float4* __restrict__ nrm, float* __restrict__ cov6, unsigned char* __restrict__ keep) {
  float a[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int r = 0; r < nf; r++) {   // warp-uniform
    const float qx = __shfl_sync(kFull, x, r), qy = __shfl_sync(kFull, y, r), qz = __shfl_sync(kFull, z, r);
    a[0] += qx * qx; a[1] += qx * qy; a[2] += qx * qz; a[3] += qy * qy; a[4] += qy * qz; a[5] += qz * qz;
    a[6] += qx; a[7] += qy; a[8] += qz;
  }
  if ((threadIdx.x & 31) != 0) return;
  float C[9], n[3], curv;
  const float NaN = __int_as_float(0x7fffffff);
  if (nf < 3) {
    n[0] = n[1] = n[2] = curv = NaN;
    for (int j = 0; j < 9; j++) C[j] = NaN;
  } else {
    const float cnt = (float)nf;
    for (int j = 0; j < 9; j++) a[j] = a[j] / cnt;
    C[0] = a[0] - a[6] * a[6]; C[1] = a[1] - a[6] * a[7]; C[2] = a[2] - a[6] * a[8];
    C[4] = a[3] - a[7] * a[7]; C[5] = a[4] - a[7] * a[8]; C[8] = a[5] - a[8] * a[8];
    C[3] = C[1]; C[6] = C[2]; C[7] = C[5];
    float lambda;
    eigen33_smallest(C, lambda, n);
    const float eig_sum = C[0] + C[4] + C[8];
    curv = eig_sum != 0.f ? fabsf(lambda / eig_sum) : 0.f;
    // flipNormalTowardsViewpoint(point, 0, 0, vpz, nx, ny, nz)
    const float vx = 0.f - p.x, vy = 0.f - p.y, vz = vpz - p.z;
    if (vx * n[0] + vy * n[1] + vz * n[2] < 0.f) { n[0] *= -1.f; n[1] *= -1.f; n[2] *= -1.f; }
  }
  nrm[i] = make_float4(n[0], n[1], n[2], curv);
  float* o = cov6 + 6 * (size_t)i;
  o[0] = C[0]; o[1] = C[1]; o[2] = C[2]; o[3] = C[4]; o[4] = C[5]; o[5] = C[8];
  // normals->at(i).getNormalVector3fMap().normalized().dot(UnitZ), |dot| > cos(normal_filter_thresh) in double
  const float z2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
  const float nz = z2 > 0.f ? n[2] / sqrtf(z2) : n[2];
  keep[i] = (double)fabsf(nz) > cos_thr ? 1 : 0;
}

__global__ void __launch_bounds__(kFloorWarps * 32) floor_normals_kernel(MapView mv, const float4* __restrict__ pts, const int* __restrict__ n_dev,
                                                                         float max_sq, float vpz, double cos_thr, float4* __restrict__ nrm,
                                                                         float* __restrict__ cov6, unsigned char* __restrict__ keep,
                                                                         int* __restrict__ nn) {
  __shared__ __align__(16) unsigned char s_list[kFloorWarps * kWarpListBytes];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpList wl = make_warp_list(s_list, warp);
  const int n = *n_dev, kneed = min(n, kFloorK);
  for (int i = blockIdx.x * kFloorWarps + warp; i < n; i += gridDim.x * kFloorWarps) {
    const float4 p = __ldg(pts + i);
    Neighbor nb;
    const int nf = knn_exact_warp<kFloorK>(mv, p.x, p.y, p.z, max_sq, wl, nb);
    if (lane == 0) nn[i] = nf;
    if (nf < kneed) continue;   // warp-uniform: floor_complete_kernel serves this point
    float x = 0.f, y = 0.f, z = 0.f;
    if (lane < nf) { const float4 q = __ldg(pts + nb.id); x = q.x; y = q.y; z = q.z; }
    floor_point_normal(x, y, z, nf, i, p, vpz, cos_thr, nrm, cov6, keep);
  }
}

// The exact 10-NN by a scan of the whole clipped cloud, for points whose grid search found fewer than min(n, 10) (all = 1: every
// point, when the map dropped points).  The K best are kept sorted across lanes 0 .. K-1 (as gicp_normals_complete_kernel).
__global__ void __launch_bounds__(kFloorWarps * 32) floor_complete_kernel(const float4* __restrict__ pts, const int* __restrict__ n_dev, int all,
                                                                          float vpz, double cos_thr, float4* __restrict__ nrm,
                                                                          float* __restrict__ cov6, unsigned char* __restrict__ keep,
                                                                          int* __restrict__ nn) {
  const int lane = threadIdx.x & 31;
  const int n = *n_dev, kneed = min(n, kFloorK);
  for (int i = blockIdx.x * kFloorWarps + (threadIdx.x >> 5); i < n; i += gridDim.x * kFloorWarps) {
    if (!all && nn[i] >= kneed) continue;   // warp-uniform
    const float4 p = __ldg(pts + i);
    float bd = 3.0e38f; int bi = 0x7fffffff;
    for (int j0 = 0; j0 < n; j0 += 32) {
      const int j = j0 + lane;
      float d2 = 3.0e38f;
      if (j < n) { const float4 a = __ldg(pts + j); d2 = dist2(p.x, p.y, p.z, a.x, a.y, a.z); }
      const float wd = __shfl_sync(kFull, bd, kFloorK - 1); const int wi = __shfl_sync(kFull, bi, kFloorK - 1);
      unsigned cand = __ballot_sync(kFull, j < n && (d2 < wd || (d2 == wd && j < wi)));
      while (cand) {
        const int src = __ffs(cand) - 1;
        cand &= cand - 1;
        const float nd = __shfl_sync(kFull, d2, src); const int ni = j0 + src;
        const bool less = bd < nd || (bd == nd && bi < ni);
        const int pos = __popc(__ballot_sync(kFull, less && lane < kFloorK));
        const float ud = __shfl_up_sync(kFull, bd, 1); const int ui = __shfl_up_sync(kFull, bi, 1);
        if (pos < kFloorK) {
          if (lane == pos) { bd = nd; bi = ni; }
          else if (lane > pos && lane < kFloorK) { bd = ud; bi = ui; }
        }
      }
    }
    float x = 0.f, y = 0.f, z = 0.f;
    if (lane < kneed) { const float4 q = __ldg(pts + bi); x = q.x; y = q.y; z = q.z; }
    if (lane == 0) nn[i] = kneed;
    floor_point_normal(x, y, z, kneed, i, p, vpz, cos_thr, nrm, cov6, keep);
  }
}

// ------------------------------------------------------------------ RANSAC (RandomSampleConsensus::computeModel)
// boost::mt19937 (== std::mt19937) twisted by one warp: entry i needs mt[i + 1] (old) and mt[i + 397 mod 624] (new once
// i >= 227, written by an earlier group of 32), so groups of 32 consecutive entries read, sync, then write.
__device__ __forceinline__ void mt_twist_warp(unsigned* mt) {
  const int lane = threadIdx.x & 31;
  for (int g = 0; g < kMtN; g += 32) {
    const int i = g + lane;
    unsigned v = 0;
    if (i < kMtN) {
      const unsigned y = (mt[i] & 0x80000000u) | (mt[(i + 1) % kMtN] & 0x7fffffffu);
      v = mt[(i + 397) % kMtN] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    __syncwarp();
    if (i < kMtN) mt[i] = v;
    __syncwarp();
  }
}
__device__ __forceinline__ unsigned mt_temper(unsigned y) {
  y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
  return y;
}

// isSampleGood / computeModelCoefficients' collinearity test: dy1dy2 = (p1 - p0) / (p2 - p0) over x, y, z
__device__ __forceinline__ bool sample_good(float4 p0, float4 p1, float4 p2) {
  const float d0 = (p1.x - p0.x) / (p2.x - p0.x), d1 = (p1.y - p0.y) / (p2.y - p0.y), d2 = (p1.z - p0.z) / (p2.z - p0.z);
  return d0 != d1 || d2 != d1;
}

// One warp.  Fills B hypotheses: per hypothesis getSamples (up to 1000 draws of three swaps each, rnd() = mt() >> 1) and
// computeModelCoefficients.  The generator and the shuffled indices carry over between batches (state in *st / shuf).
__global__ void __launch_bounds__(32) floor_sample_kernel(const float4* __restrict__ pts, const int* __restrict__ n_dev, FloorRng* __restrict__ st,
                                                          int* __restrict__ shuf, FloorHyp* __restrict__ hyp, int B, int first) {
  __shared__ unsigned s_mt[kMtN];
  const int lane = threadIdx.x & 31;
  const unsigned n = (unsigned)*n_dev;
  int pos, done, s0, s1, s2;
  if (first) {
    if (lane == 0) {
      s_mt[0] = 12345u;
      for (int i = 1; i < kMtN; i++) s_mt[i] = 1812433253u * (s_mt[i - 1] ^ (s_mt[i - 1] >> 30)) + (unsigned)i;
    }
    pos = kMtN; done = 0; s0 = 0; s1 = 1; s2 = 2;   // shuffled_indices_ = identity (written by the candidate compaction)
  } else {
    for (int i = lane; i < kMtN; i += 32) s_mt[i] = st->mt[i];
    pos = st->pos; done = st->done; s0 = st->s[0]; s1 = st->s[1]; s2 = st->s[2];
  }
  __syncwarp();
  for (int h = 0; h < B; h++) {
    FloorHyp o;
    o.idx[0] = o.idx[1] = o.idx[2] = -1; o.flag = -1; o.c[0] = o.c[1] = o.c[2] = o.c[3] = 0.f;
    if (!done) {
      bool good = false;
      for (int t = 0; t < 1000 && !good; t++) {
        int sel[3] = {s0, s1, s2};
#pragma unroll
        for (int j = 0; j < 3; j++) {
          if (pos >= kMtN) { mt_twist_warp(s_mt); pos = 0; }
          const unsigned r = mt_temper(s_mt[pos++]) >> 1;   // boost::uniform_int<>(0, INT_MAX) on mt19937
          const unsigned k = (unsigned)j + r % (n - (unsigned)j);
          if (lane == 0) {   // std::swap(shuffled_indices_[j], shuffled_indices_[k])
            if (k < 3u) { const int tmp = sel[j]; sel[j] = sel[k]; sel[k] = tmp; }
            else { const int tmp = shuf[k]; shuf[k] = sel[j]; sel[j] = tmp; }
          }
        }
        s0 = __shfl_sync(kFull, sel[0], 0); s1 = __shfl_sync(kFull, sel[1], 0); s2 = __shfl_sync(kFull, sel[2], 0);
        good = sample_good(__ldg(pts + s0), __ldg(pts + s1), __ldg(pts + s2));
      }
      if (!good) { done = 1; }
      else {
        o.idx[0] = s0; o.idx[1] = s1; o.idx[2] = s2;
        const float4 p0 = __ldg(pts + s0), p1 = __ldg(pts + s1), p2 = __ldg(pts + s2);
        if (!sample_good(p0, p1, p2)) o.flag = 0;
        else {
          o.flag = 1;
          const float ax = p1.x - p0.x, ay = p1.y - p0.y, az = p1.z - p0.z, bx = p2.x - p0.x, by = p2.y - p0.y, bz = p2.z - p0.z;
          float c[4] = {ay * bz - az * by, az * bx - ax * bz, ax * by - ay * bx, 0.f};
          const float zz = (c[0] * c[0] + c[2] * c[2]) + (c[1] * c[1] + c[3] * c[3]);   // normalize(): 4-dot, SSE order
          if (zz > 0.f) { const float s = sqrtf(zz); c[0] /= s; c[1] /= s; c[2] /= s; c[3] /= s; }
          c[3] = -1.f * ((c[0] * p0.x + c[2] * p0.z) + (c[1] * p0.y + c[3] * 1.0f));
          o.c[0] = c[0]; o.c[1] = c[1]; o.c[2] = c[2]; o.c[3] = c[3];
        }
      }
    }
    if (lane == 0) hyp[h] = o;
  }
  for (int i = lane; i < kMtN; i += 32) st->mt[i] = s_mt[i];
  if (lane == 0) { st->pos = pos; st->done = done; st->s[0] = s0; st->s[1] = s1; st->s[2] = s2; }
}

// countWithinDistance of every hypothesis of the batch over every candidate: integer counts, so the order of the additions
// does not matter.  The last block publishes the rows (count, flag, coefficients) to mapped host memory and clears the counts.
constexpr int kScorePts = 4;
__global__ void __launch_bounds__(kFloorBlock) floor_score_kernel(const float4* __restrict__ pts, const int* __restrict__ n_dev,
                                                                  const FloorHyp* __restrict__ hyp, int B, double threshold,
                                                                  int* __restrict__ counts, unsigned* __restrict__ done,
                                                                  FloorRow* __restrict__ rows) {
  extern __shared__ int s_cnt[];
  __shared__ bool s_last;
  const int n = *n_dev;
  for (int h = threadIdx.x; h < B; h += blockDim.x) s_cnt[h] = 0;
  __syncthreads();
  float4 p[kScorePts];
  bool v[kScorePts];
#pragma unroll
  for (int j = 0; j < kScorePts; j++) {
    const int i = (blockIdx.x * kScorePts + j) * kFloorBlock + threadIdx.x;
    v[j] = i < n;
    p[j] = v[j] ? __ldg(pts + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int h = 0; h < B; h++) {
    const FloorHyp& q = hyp[h];
    if (q.flag != 1) continue;   // uniform
    const float c[4] = {q.c[0], q.c[1], q.c[2], q.c[3]};
    int k = 0;
#pragma unroll
    for (int j = 0; j < kScorePts; j++) k += (v[j] && (double)fabsf(plane_dist(c, p[j])) < threshold) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(kFull, k, o);
    if ((threadIdx.x & 31) == 0 && k) atomicAdd(s_cnt + h, k);
  }
  __syncthreads();
  for (int h = threadIdx.x; h < B; h += blockDim.x) if (s_cnt[h]) atomicAdd(counts + h, s_cnt[h]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int h = threadIdx.x; h < B; h += blockDim.x) {
    FloorRow r;
    r.count = atomicExch(counts + h, 0);
    r.flag = hyp[h].flag;
    r.c[0] = hyp[h].c[0]; r.c[1] = hyp[h].c[1]; r.c[2] = hyp[h].c[2]; r.c[3] = hyp[h].c[3];
    rows[h] = r;
  }
  __threadfence_system();
  if (threadIdx.x == 0) *done = 0u;
}

// ------------------------------------------------------------------ host: the stop rule
// RandomSampleConsensus::computeModel (sample_consensus/impl/ransac.hpp, PCL 1.9.1) replayed on the hypotheses in draw order.
struct RansacReplay {
  int iterations = 0; unsigned skipped = 0;
  int best_count = -INT_MAX; long long best = -1;
  double k = 1.0, log_p = 0.0, one_over_n = 0.0;
  int max_iter = 10000; unsigned max_skip = 100000;
  long long consumed = 0;
  int stopped = 0;
  void init(int n_points, double probability, int max_iterations) {
    *this = RansacReplay();
    log_p = std::log(1.0 - probability);
    one_over_n = 1.0 / (double)n_points;
    max_iter = max_iterations;
    max_skip = (unsigned)max_iterations * 10u;
    stopped = !more();   // max_iterations = 0: the loop body never runs
  }
  // the while condition, checked before every draw: once it fails, the loop has ended after `consumed` hypotheses
  bool more() const { return (double)iterations < k && skipped < max_skip; }
  // one hypothesis (count, flag) of a loop that has not ended; returns true once it has
  bool step(int count, int flag) {
    if (stopped) return true;
    consumed++;
    if (flag < 0) { stopped = 1; return true; }   // "No samples could be selected!"
    if (flag == 0) { ++skipped; stopped = !more(); return stopped; }
    if (count > best_count) {
      best_count = count;
      best = consumed - 1;
      const double w = (double)count * one_over_n;
      double p_no = 1.0 - std::pow(w, 3.0);
      p_no = std::max(std::numeric_limits<double>::epsilon(), p_no);
      p_no = std::min(1.0 - std::numeric_limits<double>::epsilon(), p_no);
      k = log_p / std::log(p_no);
    }
    ++iterations;
    stopped = iterations > max_iter || !more();
    return stopped;
  }
};

}  // namespace lsd

using namespace lsd;

struct lsd_floor {
  lsd_floor_params_t p{};
  int device = 0;
  cudaStream_t stream = nullptr;
  lsd_voxelgrid* vg = nullptr;
  lsd_map* map = nullptr;
  size_t cap = 0;                        // points the per-point buffers hold
  float4 *d_in = nullptr, *d_pre = nullptr, *d_clip = nullptr, *d_cand = nullptr, *d_inl = nullptr;
  float4* d_nrm = nullptr; float* d_cov = nullptr; unsigned char* d_keep = nullptr; int* d_nn = nullptr; int* d_shuf = nullptr;
  void* d_chain = nullptr; size_t chain_bytes = 0;   // tickets + prefix words of the compaction chains
  int* d_counts = nullptr;               // [5] stage counts: vg, pre, clip, cand, inliers ; [8..] done counter
  FloorRng* d_rng = nullptr;
  FloorHyp* d_hyp = nullptr; size_t hyp_cap = 0;
  int* d_score = nullptr; int score_cap = 0;
  FloorRow* h_rows = nullptr; FloorRow* d_rows = nullptr; int rows_cap = 0;
  int* h_n = nullptr;                    // pinned: stage counts read back
  // last call
  lsd_floor_result_t last{};
  int n_pre = 0, n_clip = 0, n_cand = 0, n_inl = 0;
  bool pre_is_input = false;             // no prefilter: the prefiltered stage is the input
  const float4* in_used = nullptr;
  std::vector<int> h_counts, h_flags;    // replayed hypotheses, draw order
  long long launches = 0;
};

namespace lsd {

static lsd_status_t floor_reserve(lsd_floor* f, size_t n) {
  if (n <= f->cap) return LSD_OK;
  size_t c = std::max<size_t>(n, 4096);
  void* ptrs[] = {f->d_in, f->d_pre, f->d_clip, f->d_cand, f->d_inl, f->d_nrm, f->d_cov, f->d_keep, f->d_nn, f->d_shuf, f->d_chain};
  for (void* q : ptrs) cudaFree(q);
  f->cap = 0;
  f->chain_bytes = 64 * 4 + ((c + kFloorBlock - 1) / kFloorBlock + 1) * 8 * 4;
  LSD_CUDA(cudaMalloc((void**)&f->d_in, c * 16));
  LSD_CUDA(cudaMalloc((void**)&f->d_pre, c * 16));
  LSD_CUDA(cudaMalloc((void**)&f->d_clip, c * 16));
  LSD_CUDA(cudaMalloc((void**)&f->d_cand, c * 16));
  LSD_CUDA(cudaMalloc((void**)&f->d_inl, c * 16));
  LSD_CUDA(cudaMalloc((void**)&f->d_nrm, c * 16));
  LSD_CUDA(cudaMalloc((void**)&f->d_cov, c * 24));
  LSD_CUDA(cudaMalloc((void**)&f->d_keep, c));
  LSD_CUDA(cudaMalloc((void**)&f->d_nn, c * 4));
  LSD_CUDA(cudaMalloc((void**)&f->d_shuf, c * 4));
  LSD_CUDA(cudaMalloc(&f->d_chain, f->chain_bytes));
  f->cap = c;
  if (f->vg) { lsd_voxelgrid_destroy(f->vg); f->vg = nullptr; }
  if (f->p.prefilter_leaf > 0.f) {
    lsd_status_t s = lsd_voxelgrid_create(&f->vg, (int)c, 28);
    if (s) return s;
  }
  // the normals' point map: at least two lines per point
  int l2 = 12;
  while (l2 < 26 && (1ull << l2) < (unsigned long long)c * 2ull) l2++;
  if (f->map) { lsd_map_destroy(f->map); f->map = nullptr; }
  lsd_status_t s = lsd_map_create(&f->map, kFloorMapRes, l2);
  if (s) return s;
  cudaStreamDestroy(f->map->stream);
  f->map->stream = nullptr;
  return LSD_OK;
}

// chain scratch: [0] ticket words (one per chain, 4 chains), then 4 prefix arrays
static void floor_chain(lsd_floor* f, int which, unsigned** ticket, unsigned long long** prefix) {
  const size_t nb = (f->cap + kFloorBlock - 1) / kFloorBlock + 1;
  *ticket = reinterpret_cast<unsigned*>(f->d_chain) + which;
  *prefix = reinterpret_cast<unsigned long long*>(static_cast<char*>(f->d_chain) + 256) + (size_t)which * nb;
}

static lsd_status_t floor_hyp_reserve(lsd_floor* f, size_t n) {
  if (n <= f->hyp_cap) return LSD_OK;
  size_t c = std::max(n, 2 * f->hyp_cap);
  FloorHyp* nh = nullptr;
  LSD_CUDA(cudaMalloc((void**)&nh, c * sizeof(FloorHyp)));
  if (f->d_hyp) LSD_CUDA(cudaMemcpyAsync(nh, f->d_hyp, f->hyp_cap * sizeof(FloorHyp), cudaMemcpyDeviceToDevice, f->stream));
  LSD_CUDA(cudaStreamSynchronize(f->stream));
  cudaFree(f->d_hyp);
  f->d_hyp = nh; f->hyp_cap = c;
  return LSD_OK;
}

static lsd_status_t floor_run(lsd_floor* f, const float4* d_in, int n, lsd_floor_result_t* res) {
  const lsd_floor_params_t& P = f->p;
  cudaStream_t st = f->stream;
  lsd_floor_result_t r{};
  r.reason = LSD_FLOOR_EMPTY;
  r.n_input = n;
  f->n_pre = f->n_clip = f->n_cand = f->n_inl = 0;
  f->h_counts.clear(); f->h_flags.clear();
  f->launches = 0;
  f->in_used = d_in;
  f->pre_is_input = !(P.prefilter_leaf > 0.f);
  if (n == 0) { f->last = r; *res = r; return LSD_OK; }
  LSD_CUDA(cudaMemsetAsync(f->d_chain, 0, f->chain_bytes, st));
  // 1. prefilter: VoxelGrid (LSD_ERR_GRID_OVERFLOW: the input unchanged, as PCL) + the distance filter
  const float4* src = d_in;
  const int* n_src = nullptr;
  if (!f->pre_is_input) {
    float4* vg_out = f->d_inl;   // scratch until the inliers are written
    lsd_status_t s = vg_run(f->vg, d_in, n, P.prefilter_leaf, vg_out, f->d_counts, st);
    if (s) return s;
    f->launches += vg_launches(f->vg);
    src = vg_out; n_src = f->d_counts;
  }
  // 2. height clip (+ the distance filter) and the map insert of the clipped points
  LSD_CUDA(cudaMemsetAsync(f->map->view.lines, 0, f->map->n_lines * sizeof(CellLine), st));
  LSD_CUDA(cudaMemsetAsync(f->map->view.tags, 0, f->map->n_lines, st));
  LSD_CUDA(cudaMemsetAsync(f->map->view.counters, 0, 4 * sizeof(unsigned long long), st));
  unsigned* tk; unsigned long long* pf;
  floor_chain(f, 0, &tk, &pf);
  floor_clip_kernel<<<(n + kFloorBlock - 1) / kFloorBlock, kFloorBlock, 0, st>>>(
      src, n_src, n, f->pre_is_input ? 0 : 1, P.distance_near, P.distance_far, P.clip_keep_d, P.clip_cut_d,
      f->pre_is_input ? nullptr : f->d_pre, f->d_clip, f->map->view, tk, pf, f->d_counts + 1, f->d_counts + 2);
  LSD_CUDA(cudaGetLastError());
  f->launches++;
  unsigned long long* dropped_dev = f->map->view.counters + 2;
  LSD_CUDA(cudaMemcpyAsync(f->h_n, f->d_counts, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaMemcpyAsync(f->h_n + 8, dropped_dev, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  if (f->vg) LSD_CUDA(cudaMemcpyAsync(f->h_n + 12, &f->vg->grid->status, sizeof(int), cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  r.round_trips++;
  if (f->vg && f->h_n[12] == LSD_ERR_CAPACITY) { set_error("lsd_floor_detect: the prefilter grid exceeds 2^28 leaves (raise prefilter_leaf)"); return LSD_ERR_CAPACITY; }
  f->n_pre = f->pre_is_input ? n : f->h_n[1];
  f->n_clip = f->h_n[2];
  const unsigned long long dropped = *reinterpret_cast<unsigned long long*>(f->h_n + 8);
  r.n_prefiltered = f->n_pre; r.n_clipped = f->n_clip; r.map_dropped = (int)std::min<unsigned long long>(dropped, INT_MAX);
  // 3. normals + normal filter
  const double cos_nf = std::cos(P.normal_filter_deg * M_PI / 180.0);
  const float4* cand_src = f->d_clip;
  int* n_cand_dev = f->d_counts + 2;
  if (P.use_normal_filtering && f->n_clip > 0) {
    const int wg = std::max(1, std::min((f->n_clip + kFloorWarps - 1) / kFloorWarps, kNumSms * 8));
    if (dropped == 0) {
      floor_normals_kernel<<<wg, kFloorWarps * 32, 0, st>>>(f->map->view, f->d_clip, f->d_counts + 2, kFloorSearchSq, P.viewpoint_z, cos_nf,
                                                           f->d_nrm, f->d_cov, f->d_keep, f->d_nn);
      f->launches++;
    }
    floor_complete_kernel<<<wg, kFloorWarps * 32, 0, st>>>(f->d_clip, f->d_counts + 2, dropped ? 1 : 0, P.viewpoint_z, cos_nf, f->d_nrm, f->d_cov,
                                                          f->d_keep, f->d_nn);
    f->launches++;
    floor_chain(f, 1, &tk, &pf);
    floor_compact_kernel<<<(f->n_clip + kFloorBlock - 1) / kFloorBlock, kFloorBlock, 0, st>>>(f->d_clip, f->d_counts + 2, f->d_keep, nullptr, 0.0,
                                                                                            f->d_cand, f->d_shuf, tk, pf, f->d_counts + 3);
    LSD_CUDA(cudaGetLastError());
    f->launches++;
    cand_src = f->d_cand;
    n_cand_dev = f->d_counts + 3;
    LSD_CUDA(cudaMemcpyAsync(f->h_n + 3, f->d_counts + 3, sizeof(int), cudaMemcpyDeviceToHost, st));
    LSD_CUDA(cudaStreamSynchronize(st));
    r.round_trips++;
    f->n_cand = f->h_n[3];
  } else {
    f->n_cand = f->n_clip;
    if (f->n_clip > 0) {   // shuffled_indices_ = identity
      floor_chain(f, 1, &tk, &pf);
      floor_compact_kernel<<<(f->n_clip + kFloorBlock - 1) / kFloorBlock, kFloorBlock, 0, st>>>(f->d_clip, f->d_counts + 2, nullptr, nullptr, 0.0,
                                                                                              f->d_cand, f->d_shuf, tk, pf, f->d_counts + 3);
      LSD_CUDA(cudaGetLastError());
      f->launches++;
    }
    cand_src = f->d_cand;
    n_cand_dev = f->d_counts + 3;
  }
  r.n_candidates = f->n_cand;
  // 4. gate
  if (f->n_cand < P.floor_pts_thresh) { r.reason = LSD_FLOOR_FEW_CANDIDATES; goto done; }
  if (f->n_cand < 3) { r.reason = LSD_FLOOR_NO_MODEL; goto done; }   // getSamples: fewer points than a sample
  {
    // 5. RANSAC: batches of B hypotheses until the replayed stop rule ends inside a batch
    const int B = P.hypotheses_per_batch;
    RansacReplay rp;
    rp.init(f->n_cand, P.ransac_probability, P.ransac_max_iterations);
    int batch = 0;
    while (!rp.stopped) {
      lsd_status_t s = floor_hyp_reserve(f, (size_t)(batch + 1) * B);
      if (s) return s;
      FloorHyp* hb = f->d_hyp + (size_t)batch * B;
      floor_sample_kernel<<<1, 32, 0, st>>>(cand_src, n_cand_dev, f->d_rng, f->d_shuf, hb, B, batch == 0 ? 1 : 0);
      const int sg = std::max(1, (f->n_cand + kFloorBlock * kScorePts - 1) / (kFloorBlock * kScorePts));
      floor_score_kernel<<<sg, kFloorBlock, (size_t)B * sizeof(int), st>>>(cand_src, n_cand_dev, hb, B, P.ransac_threshold, f->d_score,
                                                                         reinterpret_cast<unsigned*>(f->d_counts + 8), f->d_rows);
      LSD_CUDA(cudaGetLastError());
      f->launches += 2;
      LSD_CUDA(cudaStreamSynchronize(st));
      r.round_trips++;
      batch++;
      for (int h = 0; h < B && !rp.stopped; h++) {
        const FloorRow& row = f->h_rows[h];
        const long long before = rp.consumed;
        rp.step(row.count, row.flag);
        if (rp.consumed > before) { f->h_counts.push_back(row.count); f->h_flags.push_back(row.flag); }
        if (rp.best == rp.consumed - 1 && rp.consumed > before && row.flag == 1) {
          r.coeffs[0] = row.c[0]; r.coeffs[1] = row.c[1]; r.coeffs[2] = row.c[2]; r.coeffs[3] = row.c[3];
        }
      }
    }
    r.batches = batch;
    r.hypotheses_scored = (long long)batch * B;
    r.iterations = rp.iterations;
    r.skipped = (int)rp.skipped;
    r.best_hypothesis = (int)rp.best;
    if (rp.best < 0) { r.reason = LSD_FLOOR_NO_MODEL; r.coeffs[0] = r.coeffs[1] = r.coeffs[2] = r.coeffs[3] = 0.f; goto done; }
    // selectWithinDistance of the best model: the inlier cloud, ascending index
    floor_chain(f, 2, &tk, &pf);
    floor_compact_kernel<<<(f->n_cand + kFloorBlock - 1) / kFloorBlock, kFloorBlock, 0, st>>>(cand_src, n_cand_dev, nullptr, f->d_hyp + rp.best,
                                                                                            P.ransac_threshold, f->d_inl, nullptr, tk, pf,
                                                                                            f->d_counts + 4);
    LSD_CUDA(cudaGetLastError());
    f->launches++;
    f->n_inl = rp.best_count;   // the same predicate as countWithinDistance
    r.n_inliers = rp.best_count;
    // 6. gates
    if (rp.best_count < P.floor_pts_thresh) { r.reason = LSD_FLOOR_FEW_INLIERS; goto done; }
    if ((double)std::fabs(r.coeffs[2]) < std::cos(P.floor_normal_deg * M_PI / 180.0)) { r.reason = LSD_FLOOR_NOT_VERTICAL; goto done; }
    if (r.coeffs[2] < 0.0f) for (int j = 0; j < 4; j++) r.coeffs[j] *= -1.0f;
    r.found = 1;
    r.reason = LSD_FLOOR_FOUND;
  }
done:
  LSD_CUDA(cudaStreamSynchronize(st));
  r.launches = (int)f->launches;
  f->last = r;
  *res = r;
  return LSD_OK;
}

}  // namespace lsd

extern "C" {

void lsd_floor_default_params(lsd_floor_params_t* p, int preset) {
  if (!p) return;
  *p = lsd_floor_params_t{};
  p->prefilter_leaf = 0.f;
  p->distance_near = 0.1; p->distance_far = 100.0;            // prefiltering_nodelet.cpp:81-83
  p->clip_keep_d = 1.5f; p->clip_cut_d = -1.5f;               // graph_utils.cpp:331-338
  p->use_normal_filtering = 1;
  p->normal_k = 10;
  p->normal_filter_deg = 20.0;
  p->viewpoint_z = 0.f;
  p->ransac_threshold = 0.1;
  p->ransac_probability = 0.99;                               // SampleConsensus defaults (PCL 1.9.1)
  p->ransac_max_iterations = 10000;
  p->floor_pts_thresh = 1024;
  p->floor_normal_deg = 10.0;
  p->hypotheses_per_batch = 256;
  if (preset == LSD_FLOOR_MAPPING) {
    p->prefilter_leaf = 0.2f;                                 // InitParameter::resolution of the mapping preset
    p->clip_keep_d = 2.0f; p->clip_cut_d = -1.0f;             // floor_detection_nodelet.cpp:39-41,83-84
  } else if (preset == LSD_FLOOR_RENDER) {
    p->ransac_threshold = 0.2;                                // map_render.cpp:105
  }
}

lsd_status_t lsd_floor_create(lsd_floor_t** out, const lsd_floor_params_t* p) {
  if (!out || !p) return LSD_ERR_INVALID;
  if (p->normal_k != 10 || p->hypotheses_per_batch < 1 || p->hypotheses_per_batch > kMaxHypBatch || p->ransac_max_iterations < 0 ||
      !(p->ransac_probability > 0.0 && p->ransac_probability < 1.0) || p->prefilter_leaf < 0.f) {
    set_error("lsd_floor_create: bad parameters (normal_k must be 10, 1 <= hypotheses_per_batch <= 12288, 0 < probability < 1)");
    return LSD_ERR_INVALID;
  }
  lsd_status_t s = ensure_device();
  if (s) return s;
  s = upload_stencils();
  if (s) return s;
  lsd_floor* f = new lsd_floor();
  f->p = *p;
  cudaGetDevice(&f->device);
  const int B = p->hypotheses_per_batch;
  cudaError_t e = cudaStreamCreateWithFlags(&f->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc((void**)&f->d_counts, 64 * sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(f->d_counts, 0, 64 * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc((void**)&f->d_rng, sizeof(FloorRng));
  if (e == cudaSuccess) e = cudaMalloc((void**)&f->d_score, (size_t)B * sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(f->d_score, 0, (size_t)B * sizeof(int));
  if (e == cudaSuccess) e = cudaHostAlloc((void**)&f->h_rows, (size_t)B * sizeof(FloorRow), cudaHostAllocMapped);
  if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)&f->d_rows, f->h_rows, 0);
  if (e == cudaSuccess) e = cudaHostAlloc((void**)&f->h_n, 64 * sizeof(int), cudaHostAllocDefault);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { lsd_status_t r = cuda_fail(e, "lsd_floor_create", __FILE__, __LINE__); lsd_floor_destroy(f); return r; }
  *out = f;
  return LSD_OK;
}

lsd_status_t lsd_floor_destroy(lsd_floor_t* f) {
  if (!f) return LSD_OK;
  cudaSetDevice(f->device);
  if (f->stream) cudaStreamSynchronize(f->stream);
  void* ptrs[] = {f->d_in, f->d_pre, f->d_clip, f->d_cand, f->d_inl, f->d_nrm, f->d_cov, f->d_keep, f->d_nn, f->d_shuf, f->d_chain,
                  f->d_counts, f->d_rng, f->d_hyp, f->d_score};
  for (void* q : ptrs) cudaFree(q);
  if (f->h_rows) cudaFreeHost(f->h_rows);
  if (f->h_n) cudaFreeHost(f->h_n);
  if (f->vg) lsd_voxelgrid_destroy(f->vg);
  if (f->map) lsd_map_destroy(f->map);
  if (f->stream) cudaStreamDestroy(f->stream);
  delete f;
  return LSD_OK;
}

lsd_status_t lsd_floor_detect_dev(lsd_floor_t* f, const float* xyzi_dev, int n, lsd_floor_result_t* res) {
  if (!f || !res || n < 0 || (n > 0 && !xyzi_dev)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(f->device));
  lsd_status_t s = floor_reserve(f, (size_t)n);
  if (s) return s;
  return floor_run(f, reinterpret_cast<const float4*>(xyzi_dev), n, res);
}

lsd_status_t lsd_floor_detect(lsd_floor_t* f, const float* xyzi_host, int n, lsd_floor_result_t* res) {
  if (!f || !res || n < 0 || (n > 0 && !xyzi_host)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(f->device));
  lsd_status_t s = floor_reserve(f, (size_t)n);
  if (s) return s;
  if (n > 0) LSD_CUDA(cudaMemcpyAsync(f->d_in, xyzi_host, (size_t)n * 16, cudaMemcpyHostToDevice, f->stream));
  return floor_run(f, f->d_in, n, res);
}

static lsd_status_t floor_stage(lsd_floor_t* f, int stage, const float4** src, int* n) {
  switch (stage) {
    case LSD_FLOOR_STAGE_PREFILTERED: *src = f->pre_is_input ? f->in_used : f->d_pre; *n = f->n_pre; return LSD_OK;
    case LSD_FLOOR_STAGE_CLIPPED: *src = f->d_clip; *n = f->n_clip; return LSD_OK;
    case LSD_FLOOR_STAGE_CANDIDATES: *src = f->d_cand; *n = f->n_cand; return LSD_OK;
    case LSD_FLOOR_STAGE_INLIERS: *src = f->d_inl; *n = f->n_inl; return LSD_OK;
    default: set_error("lsd_floor_get_cloud: unknown stage %d", stage); return LSD_ERR_INVALID;
  }
}

lsd_status_t lsd_floor_get_cloud_dev(lsd_floor_t* f, int stage, const float** xyzi_dev, int* n) {
  if (!f || !xyzi_dev || !n) return LSD_ERR_INVALID;
  const float4* src; lsd_status_t s = floor_stage(f, stage, &src, n);
  if (s) return s;
  LSD_CUDA(cudaStreamSynchronize(f->stream));
  *xyzi_dev = reinterpret_cast<const float*>(src);
  return LSD_OK;
}

lsd_status_t lsd_floor_get_cloud(lsd_floor_t* f, int stage, float* out, int cap, int* n) {
  if (!f || !n || cap < 0 || (cap > 0 && !out)) return LSD_ERR_INVALID;
  const float4* src; lsd_status_t s = floor_stage(f, stage, &src, n);
  if (s) return s;
  LSD_CUDA(cudaSetDevice(f->device));
  LSD_CUDA(cudaStreamSynchronize(f->stream));
  const int m = std::min(*n, cap);
  if (m > 0) LSD_CUDA(cudaMemcpy(out, src, (size_t)m * 16, cudaMemcpyDeviceToHost));
  return LSD_OK;
}

lsd_status_t lsd_floor_get_normals(lsd_floor_t* f, float* normal4, float* cov6, int cap, int* n) {
  if (!f || !n || cap < 0) return LSD_ERR_INVALID;
  *n = f->p.use_normal_filtering ? f->n_clip : 0;
  LSD_CUDA(cudaSetDevice(f->device));
  LSD_CUDA(cudaStreamSynchronize(f->stream));
  const int m = std::min(*n, cap);
  if (m > 0 && normal4) LSD_CUDA(cudaMemcpy(normal4, f->d_nrm, (size_t)m * 16, cudaMemcpyDeviceToHost));
  if (m > 0 && cov6) LSD_CUDA(cudaMemcpy(cov6, f->d_cov, (size_t)m * 24, cudaMemcpyDeviceToHost));
  return LSD_OK;
}

lsd_status_t lsd_floor_last_samples(lsd_floor_t* f, int32_t* idx3, int32_t* flags, int32_t* counts, int cap, int* n) {
  if (!f || !n || cap < 0) return LSD_ERR_INVALID;
  *n = (int)f->h_flags.size();
  const int m = std::min(*n, cap);
  if (m > 0 && idx3) {
    LSD_CUDA(cudaSetDevice(f->device));
    LSD_CUDA(cudaStreamSynchronize(f->stream));
    std::vector<FloorHyp> h((size_t)m);
    LSD_CUDA(cudaMemcpy(h.data(), f->d_hyp, (size_t)m * sizeof(FloorHyp), cudaMemcpyDeviceToHost));
    for (int i = 0; i < m; i++) for (int j = 0; j < 3; j++) idx3[3 * i + j] = h[i].idx[j];
  }
  for (int i = 0; i < m; i++) {
    if (flags) flags[i] = f->h_flags[i];
    if (counts) counts[i] = f->h_counts[i];
  }
  return LSD_OK;
}

lsd_status_t lsd_ransac_replay(const int32_t* counts, const int32_t* flags, int n, int n_points, double probability, int max_iterations,
                               int* consumed, int* best, int* iterations, int* skipped) {
  if (n < 0 || n_points < 1 || (n > 0 && (!counts || !flags)) || !consumed || !best) return LSD_ERR_INVALID;
  RansacReplay rp;
  rp.init(n_points, probability, max_iterations);
  for (int i = 0; i < n && !rp.stopped; i++) rp.step(counts[i], flags[i]);
  *consumed = rp.stopped ? (int)rp.consumed : -1;
  *best = (int)rp.best;
  if (iterations) *iterations = rp.iterations;
  if (skipped) *skipped = (int)rp.skipped;
  return LSD_OK;
}

}  // extern "C"
