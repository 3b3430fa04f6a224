// overlap.cu — the overlap detector of map merging: OverlapDetector::detect (slam/localization/include/overlap_merge.hpp:63-296,
// called from MapLoader::mergeMapSLAM, map_loader.cpp:118-137, when both maps share a GNSS origin), with its inlier
// prescreen and its NDT coarse stage batched over every (new key frame, candidate) pair of a fragment.
//
// The reference runs, per new key frame and candidate, a kd-tree inlier prescreen (calc_fitness_score, :225-263) and an
// NDT_CUDA alignment (:157-179), one after another, then a FAST_GICP of the new key frame against the best candidate
// accumulated with its graph neighbours (:185-210).  Here:
//   * overlap_filter_kernel filters every cloud of the call (:213-223) and compacts it in input order, one block per cloud;
//     each filtered target gets its exact-NN point map (build_point_map: an incomplete map sends every search to a scan
//     of the whole filtered cloud).
//   * overlap_prescreen_kernel runs calc_fitness_score of every pair in one launch: float transform in PCL's order, the
//     filter, the exact 1-NN (nn1_exact_thread / nn_scan_thread, reg.cu), integer counts and a double sum per pair.
//   * ndt_cost_pairs_kernel evaluates the next NDT cost of every live pair in one launch per Levenberg-Marquardt round,
//     each pair against its own new key frame's NDT table (the descriptor carries the NdtView, as GaCand carries the
//     VgView in galign.cu).  Per pair it is ndt_cost_batch_kernel (loop.cu): the single-pair grid, ndt_point,
//     block_partials<29> and loop_finalize's fold, so every pair has the bits of lsd_reg's single-pair kernels on the
//     same NDT table (ov_serial runs them for comparison).  The
//     fitness of the converged pairs is one fitness_pairs_kernel launch (galign.cu).
//   * overlap_accum_kernel writes the best candidate and its transformed graph neighbours into one device cloud for the
//     GICP stage (lsd_reg, sequential over the new key frames that have a best match).
// Included by lsdreg.cu after reg.cu, loop.cu and galign.cu.
#include <deque>
#include <map>
#include <set>

namespace lsd {

// One pair of a batched prescreen or NDT launch.
struct OvCand {
  NdtView ndt;           // cost: the new key frame's NDT table
  MapView mv;            // prescreen: point map of the filtered target
  NnTarget tg;           // prescreen: the filtered target cloud as the map's fallback (fitness_target)
  long long corr_off;    // cost: [n_off, n] correspondence slots at this offset of the correspondence pool
  int src_off, n;        // source cloud: first point in the key-frame pool, point count
  int blk_off, n_blk;    // first block of the launch, blocks it gets (the single-pair grid for n)
  int row;               // result row (pair index in the caller's list)
  int update, deriv;     // cost: linearize / accumulate H and b
  Pose34f lin, ev;       // cost: linearisation / evaluation pose; prescreen: ev is the pose
};

// One cloud of overlap_filter_kernel: n points at src, the kept ones written from dst on.
struct OvFilt { const float4* src; float4* dst; int n; };

// One piece of the accumulated target: n points at src written at out + dst_off, through T (row-major 3x4, double)
// unless identity (the best candidate's own cloud, appended as it is, :187).
struct OvPiece { const float4* src; int n, dst_off, identity; double T[12]; };

// filter() (:213-223): sqrtf(x*x + y*y) < range and z > min_z, in float without contraction.
__device__ __forceinline__ bool ov_keep(float x, float y, float z, float range, float min_z) {
  return sqrtf(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))) < range && z > min_z;   // IEEE sqrt (-prec-sqrt)
}

// pcl::transformPointCloud with an Eigen::Matrix4f: ((r0 x + r1 y) + r2 z) + t per row, in float, never fused.
__device__ __forceinline__ float3 ov_xform_rn(const Pose34f& T, const float4 a) {
  float o[3];
#pragma unroll
  for (int r = 0; r < 3; r++)
    o[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T.R[3 * r], a.x), __fmul_rn(T.R[3 * r + 1], a.y)), __fmul_rn(T.R[3 * r + 2], a.z)), T.t[r]);
  return make_float3(o[0], o[1], o[2]);
}

// Block b filters cloud jobs[b] into jobs[b].dst, in input order (a block-wide prefix of the warp ballots per chunk of
// blockDim.x points), and stores the kept count in counts[b].
__global__ void __launch_bounds__(1024) overlap_filter_kernel(const OvFilt* __restrict__ jobs, float range, float min_z,
                                                              int* __restrict__ counts) {
  __shared__ int s_warp[32];
  __shared__ int s_total;
  const OvFilt job = jobs[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  int base = 0;
  for (int i0 = 0; i0 < job.n; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    bool keep = false;
    if (i < job.n) { p = __ldg(job.src + i); keep = ov_keep(p.x, p.y, p.z, range, min_z); }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {
      const int v = lane < n_warps ? s_warp[lane] : 0;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
      s_warp[lane] = incl - v;
      if (lane == 31) s_total = incl;
    }
    __syncthreads();
    if (keep) job.dst[base + s_warp[warp] + __popc(bal & ((1u << lane) - 1u))] = p;
    base += s_total;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = base;
}

// calc_fitness_score(target, source, T, max_range) (:225-263) of every pair of the launch: source points transformed by
// the pair's float pose, filtered, and each kept one's exact nearest neighbour in the filtered target, counted when the
// float d2 <= the double max_range.  Row of pair c: (sum of d2, counted, kept).
__global__ void __launch_bounds__(256) overlap_prescreen_kernel(const float4* __restrict__ pool, const OvCand* __restrict__ cands,
                                                                int n_cand, float range, float min_z, float search_sq, double max_range,
                                                                double* __restrict__ partials, unsigned* __restrict__ done,
                                                                double* __restrict__ result, double seq) {
  __shared__ double s_acc[8][3];
  const int c = loop_cand_of_block(cands, n_cand);
  const int n = cands[c].n, G = cands[c].n_blk, lb = (int)blockIdx.x - cands[c].blk_off;
  const MapView mv = cands[c].mv;
  const NnTarget tg = cands[c].tg;
  const Pose34f T = cands[c].ev;
  const float4* src = pool + cands[c].src_off;
  double sum = 0.0, nr = 0.0, nf = 0.0;
  for (int i = lb * blockDim.x + threadIdx.x; i < n; i += G * blockDim.x) {
    const float3 q = ov_xform_rn(T, __ldg(src + i));
    if (!ov_keep(q.x, q.y, q.z, range, min_z)) continue;
    nf += 1.0;
    float d2 = 3.0e38f; int id;
    bool found = !tg.all && nn1_exact_thread(mv, q.x, q.y, q.z, search_sq, &d2, &id);
    if (!found && tg.pts) { d2 = nn_scan_thread(tg.pts, tg.n, q.x, q.y, q.z, &id); found = tg.n > 0; }
    if (found && (double)d2 <= max_range) { sum += (double)d2; nr += 1.0; }
  }
  sum = warp_sum(sum); nr = warp_sum(nr); nf = warp_sum(nf);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { s_acc[warp][0] = sum; s_acc[warp][1] = nr; s_acc[warp][2] = nf; }
  __syncthreads();
  if (threadIdx.x < 3) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += s_acc[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kNV + threadIdx.x] = s;
  }
  loop_finalize<3>(partials + (size_t)cands[c].blk_off * kNV, G, done + 1 + c, done, n_cand,
                   result + (size_t)(1 + cands[c].row) * kNV, result, seq);
}

// One NDT cost evaluation for every pair of the launch, each against its own new key frame's NDT table.  The body of
// ndt_cost_batch_kernel (loop.cu) with the table taken from the descriptor.
__global__ void __launch_bounds__(256) ndt_cost_pairs_kernel(const float4* __restrict__ pool, const OvCand* __restrict__ cands,
                                                             int n_cand, int n_off, int* __restrict__ corr_pool, double* __restrict__ partials,
                                                             unsigned* __restrict__ done, double* __restrict__ result, double seq) {
  const int c = loop_cand_of_block(cands, n_cand);
  const int n = cands[c].n, G = cands[c].n_blk, lb = (int)blockIdx.x - cands[c].blk_off;
  const bool update = cands[c].update != 0, deriv = cands[c].deriv != 0;
  const NdtView v = cands[c].ndt;
  const Pose34f lin = cands[c].lin, ev = cands[c].ev;
  const float4* src = pool + cands[c].src_off;
  int* corr = corr_pool + cands[c].corr_off;
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = lb * blockDim.x + threadIdx.x; i < n; i += G * blockDim.x)
    ndt_point(v, __ldg(src + i), i, n, n_off, lin, ev, corr, update, deriv, vals);
  block_partials<29>(vals, partials);
  loop_finalize<29>(partials + (size_t)cands[c].blk_off * kNV, G, done + 1 + c, done, n_cand,
                    result + (size_t)(1 + cands[c].row) * kNV, result, seq);
}

// The accumulated target (:186-194): piece blockIdx.y, points strided over blockIdx.x.  A transformed point is
// ((T0 x + T1 y) + T2 z) + T3 per row in double (pcl::transformPointCloud with an Eigen::Matrix4d), stored as float;
// intensity copied.
__global__ void __launch_bounds__(256) overlap_accum_kernel(const OvPiece* __restrict__ pieces, float4* __restrict__ out) {
  const OvPiece& pc = pieces[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pc.n; i += gridDim.x * blockDim.x) {
    const float4 a = __ldg(pc.src + i);
    float4 o = a;
    if (!pc.identity) {
      const double x = a.x, y = a.y, z = a.z;
      const double* T = pc.T;
      o.x = (float)(((T[0] * x + T[1] * y) + T[2] * z) + T[3]);   // the library is built with -fmad=false: never fused
      o.y = (float)(((T[4] * x + T[5] * y) + T[6] * z) + T[7]);
      o.z = (float)(((T[8] * x + T[9] * y) + T[10] * z) + T[11]);
    }
    out[pc.dst_off + i] = o;
  }
}

}  // namespace lsd

// ==================================================================== host side
struct lsd_overlap {
  lsd_overlap_params_t p{};
  int device = 0;
  lsd_reg* ndt = nullptr;    // coarse stage: owns the stream and the scratch of the table builds
  lsd_reg* gicp = nullptr;   // finetune (FAST_GICP, max-corr 0.5 m, transformation epsilon 0.001)
  // key-frame pool: every cloud once, [sum n, 4] float
  float4* d_pool = nullptr; size_t pool_n = 0, pool_cap = 0;
  std::vector<size_t> kf_off;
  std::vector<int> kf_n;
  std::vector<int32_t> kf_id;
  // The tables of a slot used as a target: NDT table and point map of the cloud (coarse stage), the filtered cloud and
  // its point map (prescreen).  A slot takes a Target from `targets` on its first use as a target; lsd_overlap_detect
  // hands them all back when it returns (ov_release_targets), so the next call reuses their buffers.  Device memory is
  // bounded by the most targets one call holds (the new key frames of a fragment), not by the key frames of a merge.
  struct Target {
    lsd::NdtView ndt{}; unsigned long long ndt_lines = 0;
    lsd_map* map = nullptr;
    float4* d_filt = nullptr; size_t filt_cap = 0; int n_filt = 0; lsd_map* fmap = nullptr;
    bool ndt_built = false, filt_built = false;
    const lsd_map* filt_map() const { return n_filt > 0 ? fmap : nullptr; }   // none for an empty filtered cloud
  };
  std::deque<Target> targets;      // buffers, never moved (std::deque keeps references on push_back)
  std::vector<int> tgt_of;         // per slot: index into targets, -1 while the slot holds none
  std::vector<int> free_targets;   // indices into targets not held by a slot
  // accumulated target of the finetune, its filtered copy and that copy's point map
  float4* d_accum = nullptr; size_t accum_cap = 0;
  float4* d_accf = nullptr; size_t accf_cap = 0;
  lsd_map* accf_map = nullptr;
  int n_accum = 0, n_accf = 0;
  // small launch inputs (filter jobs, pieces) and outputs (kept counts)
  lsd::OvFilt* d_jobs = nullptr; size_t jobs_cap = 0;
  int* d_counts = nullptr; size_t counts_cap = 0;
  lsd::OvPiece* d_pieces = nullptr; size_t pieces_cap = 0;
  // batch scratch, grown to the largest batch seen
  lsd::BatchScratch<lsd::OvCand> b;
  lsd::BatchScratch<lsd::GaCand> bf;
  int* d_corr = nullptr; size_t corr_cap = 0;
  // last lsd_overlap_match / batch of lsd_overlap_detect
  std::vector<lsd::LmState> lm;
  std::vector<double> fitness;
  std::vector<lsd_overlap_report_t> reports;
  long long last_launches = 0; int last_rounds = 0;
};

namespace lsd {

constexpr int kOvKnn = 10;   // nearestKSearch(search_point, 10, ...) (:120-122)

// find_candidates' 10-NN over the key frames' translations (:67-78, :116-122): float points from the double poses, float
// squared distance ((dx dx + dy dy) + dz dz), the k = min(10, n_kf) nearest by ascending (distance, position in keyframes).
static void ov_knn(const double* poses16, const int32_t* kfs, int n_kf, int32_t new_slot, std::vector<std::pair<float, int>>& hits) {
  hits.clear();
  const double* Tn = poses16 + 16 * (size_t)new_slot;
  const float qx = (float)Tn[3], qy = (float)Tn[7], qz = (float)Tn[11];
  for (int i = 0; i < n_kf; i++) {
    const double* T = poses16 + 16 * (size_t)kfs[i];
    const float dx = (float)T[3] - qx, dy = (float)T[7] - qy, dz = (float)T[11] - qz;
    const float dxx = dx * dx, dyy = dy * dy, dzz = dz * dz;
    hits.push_back({(dxx + dyy) + dzz, i});
  }
  const size_t k = std::min((size_t)kOvKnn, hits.size());
  std::partial_sort(hits.begin(), hits.begin() + k, hits.end());
  hits.resize(k);
}

using ConnMap = std::map<int, std::set<int>>;

// graph edges -> connection_map (:80-91)
static ConnMap ov_connections(const int32_t* edges, int n_e) {
  ConnMap m;
  for (int e = 0; e < n_e; e++) { m[edges[2 * e]].insert(edges[2 * e + 1]); m[edges[2 * e + 1]].insert(edges[2 * e]); }
  return m;
}

// get_connection_count (:265-296).  The reference's queue marks a node visited when it pops it, so a node can enter the
// next level again from a later node of its own level; that can add a level when the target is not reached.  The next
// level's distinct nodes, in first-push order, do not depend on those repeats (a repeated pop pushes a subset of what
// its first pop pushed), so each level is kept without them.
static int ov_connection_count(const ConnMap& conn, int source, int target, int max_count) {
  static const std::set<int> kNone;
  std::set<int> visited;
  std::vector<int> level{source}, next;
  int count = 0;
  while (!level.empty()) {
    next.clear();
    std::set<int> in_next;
    for (int curr : level) {
      if (curr == target) return count;
      visited.insert(curr);
      auto it = conn.find(curr);
      for (int adj : it == conn.end() ? kNone : it->second)
        if (!visited.count(adj) && in_next.insert(adj).second) next.push_back(adj);
    }
    level.swap(next);
    count++;
    if (max_count > 0 && count >= max_count) break;
  }
  return count;
}

// find_candidates (:113-145): slots, in the order of the 10-NN hits.
static void ov_find(const lsd_overlap_params_t& p, const double* poses16, const int32_t* ids, const int32_t* kfs, int n_kf,
                    const ConnMap& conn, int32_t new_slot, std::vector<int32_t>& out) {
  out.clear();
  std::vector<std::pair<float, int>> hits;
  ov_knn(poses16, kfs, n_kf, new_slot, hits);
  const int new_id = ids[new_slot];
  auto own = conn.find(new_id);
  for (const auto& h : hits) {
    const int32_t k = kfs[h.second];
    if (ids[k] == new_id) continue;                                           // same key frame (:124-127)
    if (own != conn.end() && own->second.count(ids[k])) continue;             // already connected (:128-131)
    if ((double)h.first < p.distance_thresh * p.distance_thresh &&
        ov_connection_count(conn, new_id, ids[k], p.candidate_link_dist) >= p.candidate_link_dist)
      out.push_back(k);
    if ((int)out.size() >= p.max_candidate_num) break;
  }
}

// (new->mOdom.inverse() * cand->mOdom).matrix().cast<float>() (:159): Isometry3d inverse (R^T, -(R^T t)) and product
// (R_a R_b, R_a t_b + t_a), every sum left to right, then each element rounded to float.
static void ov_guess(const double* Tn, const double* Tc, float* G) {
  double Ri[9], ti[3];
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) Ri[3 * a + b] = Tn[4 * b + a];
  for (int a = 0; a < 3; a++) ti[a] = -((Ri[3 * a] * Tn[3] + Ri[3 * a + 1] * Tn[7]) + Ri[3 * a + 2] * Tn[11]);
  for (int i = 0; i < 16; i++) G[i] = 0.f;
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) G[4 * a + b] = (float)((Ri[3 * a] * Tc[b] + Ri[3 * a + 1] * Tc[4 + b]) + Ri[3 * a + 2] * Tc[8 + b]);
    G[4 * a + 3] = (float)(((Ri[3 * a] * Tc[3] + Ri[3 * a + 1] * Tc[7]) + Ri[3 * a + 2] * Tc[11]) + ti[a]);
  }
  G[15] = 1.f;
}

// Eigen::Isometry3f(M).inverse().matrix() (:198), in float: R^T and -(R^T t), sums left to right.
static void ov_inverse_f(const float* M, float* G) {
  for (int i = 0; i < 16; i++) G[i] = 0.f;
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) G[4 * a + b] = M[4 * b + a];
    const float s0 = M[a] * M[3], s1 = M[4 + a] * M[7], s2 = M[8 + a] * M[11];
    G[4 * a + 3] = -((s0 + s1) + s2);
  }
  G[15] = 1.f;
}

static void pose_f(const float* T16, Pose34f* f) {
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) f->R[3 * a + b] = T16[4 * a + b];
    f->t[a] = T16[4 * a + 3];
  }
}

static bool ov_slots_ok(const lsd_overlap* h, const int32_t* s, int n) {
  for (int i = 0; i < n; i++) if (s[i] < 0 || s[i] >= (int32_t)h->kf_n.size()) return false;
  return true;
}

// Filters the clouds jobs[0, n) in one launch (input order kept); counts[i] = points kept of job i.
static lsd_status_t ov_filter(lsd_overlap* h, const std::vector<OvFilt>& jobs, std::vector<int>& counts, long long* launches) {
  const size_t n = jobs.size();
  counts.assign(n, 0);
  if (n == 0) return LSD_OK;
  cudaStream_t st = h->ndt->stream;
  lsd_status_t s = grow_dev(h->d_jobs, h->jobs_cap, n);
  if (!s) s = grow_dev(h->d_counts, h->counts_cap, n);
  if (s) return s;
  LSD_CUDA(cudaMemcpyAsync(h->d_jobs, jobs.data(), n * sizeof(OvFilt), cudaMemcpyHostToDevice, st));
  overlap_filter_kernel<<<(unsigned)n, 1024, 0, st>>>(h->d_jobs, (float)h->p.filter_range, h->p.filter_min_z, h->d_counts);
  LSD_CUDA(cudaGetLastError());
  (*launches)++;
  LSD_CUDA(cudaMemcpyAsync(counts.data(), h->d_counts, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  return LSD_OK;
}

// The point map of a filtered cloud (build_point_map: incomplete when it refused points); none for an empty cloud.
static lsd_status_t ov_point_map(lsd_overlap* h, lsd_map** mp, const float4* pts, int n, long long* launches) {
  if (n == 0) return LSD_OK;
  lsd_status_t s = build_point_map(h->ndt, mp, pts, n);
  if (s) return s;
  (*launches)++;
  return LSD_OK;
}

// The Target of slot `slot`: its own, else one from the free set (its buffers kept for reuse), else a new one.
static lsd_overlap::Target& ov_target(lsd_overlap* h, int slot) {
  int& k = h->tgt_of[slot];
  if (k < 0) {
    if (!h->free_targets.empty()) { k = h->free_targets.back(); h->free_targets.pop_back(); }
    else { k = (int)h->targets.size(); h->targets.emplace_back(); }
    lsd_overlap::Target& t = h->targets[k];
    t.ndt_built = t.filt_built = false; t.n_filt = 0;
  }
  return h->targets[k];
}

// Every slot's Target back to the free set: the tables are rebuilt on the slot's next use as a target.
static void ov_release_targets(lsd_overlap* h) {
  for (int& k : h->tgt_of) {
    if (k < 0) continue;
    h->free_targets.push_back(k);
    k = -1;
  }
}

// The filtered copies and their point maps of the slots `slots` that have none yet: one filter launch for all of them.
static lsd_status_t ov_filtered_targets(lsd_overlap* h, const std::vector<int>& slots, long long* launches) {
  std::vector<int> todo;
  std::vector<OvFilt> jobs;
  for (int sl : slots) {
    lsd_overlap::Target& t = ov_target(h, sl);
    if (t.filt_built || std::find(todo.begin(), todo.end(), sl) != todo.end()) continue;
    lsd_status_t s = grow_dev(t.d_filt, t.filt_cap, (size_t)h->kf_n[sl]);
    if (s) return s;
    todo.push_back(sl);
    jobs.push_back(OvFilt{h->d_pool + h->kf_off[sl], t.d_filt, h->kf_n[sl]});
  }
  std::vector<int> counts;
  lsd_status_t s = ov_filter(h, jobs, counts, launches);
  if (s) return s;
  for (size_t i = 0; i < todo.size(); i++) {
    lsd_overlap::Target& t = ov_target(h, todo[i]);
    t.n_filt = counts[i];
    s = ov_point_map(h, &t.fmap, t.d_filt, t.n_filt, launches);
    if (s) return s;
    t.filt_built = true;
  }
  return LSD_OK;
}

// registration->setInputTarget(new_keyframe->mPoints) (:157) once per slot: the NDT table (the steps of
// lsd_reg_set_target_dev) and the cloud's point map (getFitnessScore, :171).
static lsd_status_t ov_ndt_target(lsd_overlap* h, int slot, long long* launches) {
  lsd_overlap::Target& t = ov_target(h, slot);
  if (t.ndt_built) return LSD_OK;
  lsd_reg* r = h->ndt;
  cudaStream_t st = r->stream;
  const float4* pts = h->d_pool + h->kf_off[slot];
  const int n = h->kf_n[slot];
  t.ndt.res = (float)r->p.resolution;
  const long long l0 = r->launches;
  lsd_status_t s = build_voxel_table<NdtBuildLine>(r, n, "NDT", t.ndt, t.ndt_lines,
      [&](NdtBuildLine* build, unsigned long long mask, unsigned* d_fail) {
        ndt_accum_kernel<<<(n + 255) / 256, 256, 0, st>>>(build, mask, t.ndt.res, pts, n, d_fail, r->sc.rank, r->sc.world, r->shard_tile);
      },
      [&](const NdtBuildLine* build, unsigned long long lines, unsigned* d_vox) {
        ndt_finalize_kernel<<<(unsigned)((lines + 255) / 256), 256, 0, st>>>(build, t.ndt.lines, lines, d_vox);
      });
  *launches += r->launches - l0;
  if (s) return s;
  s = ov_point_map(h, &t.map, pts, n, launches);
  if (s) return s;
  t.ndt_built = true;
  return LSD_OK;
}

// One pair of calc_fitness_score: source slot `src` (or the pool offset) at the float pose T against a filtered target.
struct OvScreen { int src_slot; const float4* tgt_pts; int tgt_n; const lsd_map* tgt_map; float T[16]; };

// calc_fitness_score of every pair in one launch: rows (sum, nr, n_filtered) into sum / nr / nf.
static lsd_status_t ov_prescreen(lsd_overlap* h, const std::vector<OvScreen>& q, double max_range, std::vector<double>& sum,
                                 std::vector<double>& nr, std::vector<double>& nf, long long* launches) {
  const int n = (int)q.size();
  sum.assign(n, 0.0); nr.assign(n, 0.0); nf.assign(n, 0.0);
  if (n == 0) return LSD_OK;
  size_t rows = 0;
  for (int i = 0; i < n; i++) rows += (size_t)reg_grid(h->kf_n[q[i].src_slot]);
  lsd_status_t s = h->b.reserve(n, rows);
  if (s) return s;
  const double res = h->ndt->p.map_resolution;
  int blocks = 0;
  for (int j = 0; j < n; j++) {
    const OvScreen& e = q[j];
    OvCand& c = h->b.h_cand[j];
    memset(&c, 0, sizeof(c));
    if (e.tgt_map) {
      c.mv = e.tgt_map->view;
      c.tg = fitness_target(e.tgt_map, e.tgt_pts, e.tgt_n, max_range, res);
    } else {
      c.tg = NnTarget{nullptr, 0, 1};   // empty filtered target: no search, nothing counted, the kept points still counted
    }
    c.src_off = (int)h->kf_off[e.src_slot]; c.n = h->kf_n[e.src_slot]; c.row = j;
    c.n_blk = reg_grid(c.n); c.blk_off = blocks; blocks += c.n_blk;
    pose_f(e.T, &c.ev);
  }
  cudaStream_t st = h->ndt->stream;
  double seq = 0;
  s = h->b.upload(n, st, &seq);
  if (s) return s;
  overlap_prescreen_kernel<<<blocks, 256, 0, st>>>(h->d_pool, h->b.d_cand, n, (float)h->p.filter_range, h->p.filter_min_z,
                                                   fitness_search_sq(max_range, res), max_range, h->b.d_partials, h->b.d_done, h->b.d_res, seq);
  LSD_CUDA(cudaGetLastError());
  (*launches)++;
  s = h->b.wait(st, seq);
  if (s) return s;
  for (int j = 0; j < n; j++) {
    const double* row = h->b.row(j);
    sum[j] = row[0]; nr[j] = row[1]; nf[j] = row[2];
  }
  return LSD_OK;
}

// (score, inlier ratio) as calc_fitness_score returns them (:259-262)
static void ov_score(double sum, double nr, double nf, double* score, double* ratio) {
  *score = nr > 0 ? sum / nr : DBL_MAX;
  *ratio = nr > 0 ? nr / nf : 0.0;
}

// The coarse stage of pairs (new_slots[i] target, cand[i] source) from guesses (double [n,16]): every pair's LM loop of
// lsd_reg_align, advanced together (one ndt_cost_pairs_kernel launch per round), then getFitnessScore(max_range) of the
// converged pairs in one launch.  Results in h->lm, h->fitness (DBL_MAX where not converged).
static lsd_status_t ov_coarse(lsd_overlap* h, const std::vector<int>& new_slots, const std::vector<int>& cand, const double* guesses,
                              long long* launches, int* rounds) {
  const int n = (int)cand.size();
  h->lm.assign(n, LmState());
  h->fitness.assign(n, DBL_MAX);
  if (n == 0) return LSD_OK;
  for (int i = 0; i < n; i++) {
    lsd_status_t s = ov_ndt_target(h, new_slots[i], launches);
    if (s) return s;
  }
  lsd_reg* r = h->ndt;
  const int n_off = r->p.ndt_neighbors;
  size_t rows = 0, corr = 0;
  std::vector<long long> corr_off(n);
  for (int i = 0; i < n; i++) {
    const int v = h->kf_n[cand[i]];
    rows += (size_t)std::max(reg_grid(v), warp_grid(v));
    corr_off[i] = (long long)corr;
    corr += (size_t)n_off * v;
  }
  lsd_status_t s = h->b.reserve(n, rows);
  if (!s) s = h->bf.reserve(n, rows);
  if (!s) s = grow_dev(h->d_corr, h->corr_cap, corr);
  if (s) return s;
  for (int i = 0; i < n; i++) lm_begin(h->lm[i], h->p.coarse, guesses + 16 * (size_t)i);
  cudaStream_t st = r->stream;
  for (;;) {
    int na = 0, blocks = 0;
    for (int i = 0; i < n; i++) {
      const LmState& m = h->lm[i];
      if (m.done) continue;
      OvCand& c = h->b.h_cand[na++];
      memset(&c, 0, sizeof(c));
      c.ndt = ov_target(h, new_slots[i]).ndt;
      c.src_off = (int)h->kf_off[cand[i]]; c.n = h->kf_n[cand[i]]; c.row = i;
      c.n_blk = reg_grid(c.n); c.blk_off = blocks; blocks += c.n_blk;
      c.corr_off = corr_off[i];
      c.update = m.want_update; c.deriv = m.want_update;
      T_to_pose(m.want_T, nullptr, &c.ev);
      c.lin = c.ev;   // read only when update (the linearisation pose is the evaluation pose then)
    }
    if (na == 0) break;
    double seq = 0;
    s = h->b.upload(na, st, &seq);
    if (s) return s;
    ndt_cost_pairs_kernel<<<blocks, 256, 0, st>>>(h->d_pool, h->b.d_cand, na, n_off, h->d_corr, h->b.d_partials, h->b.d_done, h->b.d_res, seq);
    LSD_CUDA(cudaGetLastError());
    (*launches)++; (*rounds)++;
    s = h->b.wait(st, seq);
    if (s) return s;
    for (int i = 0; i < n; i++) {
      LmState& m = h->lm[i];
      if (m.done) continue;
      const double* res = h->b.row(i);
      double H[36], b[6];
      if (m.want_update) unpack_hb(res, H, b);
      lm_feed(m, H, b, res[27]);
    }
  }
  // getFitnessScore(fitness_score_max_range) (:171) of the converged pairs against their new key frame's cloud
  const double max_range = h->p.fitness_score_max_range, mres = r->p.map_resolution;
  std::vector<int> conv;
  int blocks = 0;
  for (int i = 0; i < n; i++) {
    if (!h->lm[i].converged) continue;
    GaCand& c = h->bf.h_cand[conv.size()];
    memset(&c, 0, sizeof(c));
    const int t = new_slots[i];
    const lsd_map* tm = ov_target(h, t).map;
    c.mv = tm->view;
    c.tg = fitness_target(tm, h->d_pool + h->kf_off[t], h->kf_n[t], max_range, mres);
    c.src_off = (int)h->kf_off[cand[i]]; c.n = h->kf_n[cand[i]]; c.row = (int)conv.size();
    c.warp_shape = c.n < kThreadShapeMin;
    c.n_blk = c.warp_shape ? warp_grid(c.n) : reg_grid(c.n);
    c.blk_off = blocks; blocks += c.n_blk;
    T_to_pose(h->lm[i].x0, nullptr, &c.Tf);
    conv.push_back(i);
  }
  if (conv.empty()) return LSD_OK;
  double seq = 0;
  s = h->bf.upload((int)conv.size(), st, &seq);
  if (s) return s;
  fitness_pairs_kernel<<<blocks, kRegWarps * 32, 0, st>>>(h->d_pool, h->bf.d_cand, (int)conv.size(), fitness_search_sq(max_range, mres),
                                                          max_range, h->bf.d_partials, h->bf.d_done, h->bf.d_res, seq);
  LSD_CUDA(cudaGetLastError());
  (*launches)++;
  s = h->bf.wait(st, seq);
  if (s) return s;
  for (size_t j = 0; j < conv.size(); j++) {
    const double sm = h->bf.row((int)j)[0], cnt = h->bf.row((int)j)[1];
    h->fitness[conv[j]] = cnt > 0 ? sm / cnt : DBL_MAX;
  }
  return LSD_OK;
}

// The same pairs one after another through lsd_reg_align's and lsd_reg_fitness's single-pair kernels on this handle's
// tables (the coarse handle pointed at them for the call, as GaBind does in galign.cu): the bit-exactness reference of
// ov_coarse on identical tables.  *rounds = cost evaluations, one launch each.
static lsd_status_t ov_serial(lsd_overlap* h, const std::vector<int>& new_slots, const std::vector<int>& cand, const double* guesses,
                              long long* launches, int* rounds) {
  const int n = (int)cand.size();
  h->lm.assign(n, LmState());
  h->fitness.assign(n, DBL_MAX);
  lsd_reg* r = h->ndt;
  size_t corr = 0;
  for (int i = 0; i < n; i++) {
    lsd_status_t s = ov_ndt_target(h, new_slots[i], launches);
    if (s) return s;
    corr = std::max(corr, (size_t)r->p.ndt_neighbors * h->kf_n[cand[i]]);
  }
  lsd_status_t s = grow_dev(h->d_corr, h->corr_cap, corr);
  if (s) return s;
  for (int i = 0; i < n; i++) {
    const lsd_overlap::Target& t = ov_target(h, new_slots[i]);
    r->d_src = h->d_pool + h->kf_off[cand[i]]; r->n_src = h->kf_n[cand[i]];
    r->d_tgt = h->d_pool + h->kf_off[new_slots[i]]; r->n_tgt = h->kf_n[new_slots[i]];
    r->ndt = t.ndt; r->tgt_map = t.map; r->tgt_map_built = true; r->d_corr = h->d_corr;
    const long long c0 = r->launches;
    s = reg_align(r, guesses + 16 * (size_t)i);
    if (s >= 0) {
      *rounds += (int)(r->launches - c0);
      LmState& m = h->lm[i];
      memcpy(m.x0, r->final_T, sizeof(m.x0));
      m.converged = r->converged; m.iterations = r->iterations; m.iter_log = r->iter_log;
      s = m.converged ? lsd_reg_fitness(r, nullptr, h->p.fitness_score_max_range, &h->fitness[i]) : LSD_OK;
    }
    *launches += r->launches - c0;
    r->d_src = nullptr; r->n_src = 0; r->d_tgt = nullptr; r->n_tgt = 0;   // the pool and the targets own these
    r->ndt = NdtView{}; r->tgt_map = nullptr; r->tgt_map_built = false; r->d_corr = nullptr;
    if (s < 0) return s;
  }
  return LSD_OK;
}

// accum_points (:186-194): best's cloud, then for each id connected to best (ascending) the cloud of
// keyframes[keyframe_id_map[id]] under best^-1 * frame.  keyframe_id_map[id] inserts 0 for an id outside keyframes, so
// such a connection contributes keyframes[0].  Written to h->d_accum in one launch; h->n_accum = its size.
static lsd_status_t ov_accumulate(lsd_overlap* h, const double* poses16, const int32_t* kfs, int n_kf, const std::map<int, int>& id_index,
                                  const ConnMap& conn, int best, long long* launches) {
  std::vector<OvPiece> pieces;
  OvPiece p0;
  memset(&p0, 0, sizeof(p0));
  p0.src = h->d_pool + h->kf_off[best]; p0.n = h->kf_n[best]; p0.identity = 1;
  pieces.push_back(p0);
  size_t total = (size_t)p0.n;
  auto it = conn.find(h->kf_id[best]);
  if (it != conn.end() && n_kf > 0) {
    const double* Tb = poses16 + 16 * (size_t)best;
    // best->mOdom.inverse(): R^T, -(R^T t)
    double Ri[9], ti[3];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) Ri[3 * a + b] = Tb[4 * b + a];
    for (int a = 0; a < 3; a++) ti[a] = -((Ri[3 * a] * Tb[3] + Ri[3 * a + 1] * Tb[7]) + Ri[3 * a + 2] * Tb[11]);
    for (int id : it->second) {
      auto f = id_index.find(id);
      const int k = kfs[f == id_index.end() ? 0 : f->second];
      const double* Tk = poses16 + 16 * (size_t)k;
      OvPiece pc;
      memset(&pc, 0, sizeof(pc));
      pc.src = h->d_pool + h->kf_off[k]; pc.n = h->kf_n[k]; pc.dst_off = (int)total;
      for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) pc.T[4 * a + b] = (Ri[3 * a] * Tk[b] + Ri[3 * a + 1] * Tk[4 + b]) + Ri[3 * a + 2] * Tk[8 + b];
        pc.T[4 * a + 3] = ((Ri[3 * a] * Tk[3] + Ri[3 * a + 1] * Tk[7]) + Ri[3 * a + 2] * Tk[11]) + ti[a];
      }
      pieces.push_back(pc);
      total += (size_t)pc.n;
    }
  }
  if (total > (size_t)INT32_MAX) { set_error("lsd_overlap_detect: accumulated target above 2^31 points"); return LSD_ERR_CAPACITY; }
  cudaStream_t st = h->ndt->stream;
  lsd_status_t s = grow_dev(h->d_accum, h->accum_cap, total);
  if (!s) s = grow_dev(h->d_pieces, h->pieces_cap, pieces.size());
  if (s) return s;
  LSD_CUDA(cudaMemcpyAsync(h->d_pieces, pieces.data(), pieces.size() * sizeof(OvPiece), cudaMemcpyHostToDevice, st));
  int max_n = 0;
  for (const OvPiece& pc : pieces) max_n = std::max(max_n, pc.n);
  const dim3 grid((unsigned)std::max(1, std::min((max_n + 255) / 256, 64)), (unsigned)pieces.size());
  overlap_accum_kernel<<<grid, 256, 0, st>>>(h->d_pieces, h->d_accum);
  LSD_CUDA(cudaGetLastError());
  (*launches)++;
  LSD_CUDA(cudaStreamSynchronize(st));
  h->n_accum = (int)total;
  return LSD_OK;
}

}  // namespace lsd

using namespace lsd;

extern "C" {

void lsd_overlap_default_params(lsd_overlap_params_t* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->distance_thresh = 30.0;               // overlap_merge.hpp:46-51
  p->candidate_link_dist = 10;
  p->max_candidate_num = 3;
  p->fitness_score_max_range = 25.0;
  p->fitness_score_thresh = 1.5;
  p->fitness_inlier_thresh = 0.2;
  p->inlier_max_range = 1.0;               // calc_fitness_score(..., 1.0) (:160)
  p->filter_range = 100.0;                 // pointcloud_range, pointcloud_min_z (:226-227)
  p->filter_min_z = 0.5f;
  lsd_reg_default_params(&p->coarse, LSD_REG_NDT_P2D);   // select_registration_method("NDT_CUDA") (:54)
  lsd_reg_default_params(&p->accurate, LSD_REG_GICP);    // select_registration_method("FAST_GICP") (:58-60)
  p->accurate.max_corr_dist = 0.5;
  p->accurate.transformation_epsilon = 0.001;
}

lsd_status_t lsd_overlap_create(lsd_overlap_t** out, const lsd_overlap_params_t* p) {
  if (!out || !p) return LSD_ERR_INVALID;
  if (p->coarse.kind != LSD_REG_NDT_P2D || p->accurate.kind != LSD_REG_GICP) {
    set_error("lsd_overlap_create: the coarse stage is NDT_P2D, the finetune GICP");
    return LSD_ERR_INVALID;
  }
  if (p->coarse.max_process_time_us != 0) { set_error("lsd_overlap_create: the coarse stage has no timeout (overlap_merge.hpp:54)"); return LSD_ERR_INVALID; }
  if (p->max_candidate_num < 1 || p->candidate_link_dist < 0) { set_error("lsd_overlap_create: max_candidate_num >= 1, candidate_link_dist >= 0"); return LSD_ERR_INVALID; }
  lsd_overlap* h = new lsd_overlap();
  h->p = *p;
  lsd_status_t s = lsd_reg_create(&h->ndt, &p->coarse);
  if (!s) s = lsd_reg_create(&h->gicp, &p->accurate);
  if (s) { lsd_overlap_destroy(h); return s; }
  h->device = h->ndt->device;
  *out = h;
  return LSD_OK;
}

lsd_status_t lsd_overlap_destroy(lsd_overlap_t* h) {
  if (!h) return LSD_OK;
  if (h->ndt) { cudaSetDevice(h->ndt->device); cudaStreamSynchronize(h->ndt->stream); }
  for (lsd_overlap::Target& t : h->targets) {
    cudaFree(t.ndt.lines); cudaFree(t.d_filt);
    if (t.map) lsd_map_destroy(t.map);
    if (t.fmap) lsd_map_destroy(t.fmap);
  }
  if (h->accf_map) lsd_map_destroy(h->accf_map);
  cudaFree(h->d_pool); cudaFree(h->d_corr); cudaFree(h->d_accum); cudaFree(h->d_accf);
  cudaFree(h->d_jobs); cudaFree(h->d_counts); cudaFree(h->d_pieces);
  h->b.release(); h->bf.release();
  lsd_reg_destroy(h->ndt);
  lsd_reg_destroy(h->gicp);
  delete h;
  return LSD_OK;
}

lsd_status_t lsd_overlap_add_keyframe(lsd_overlap_t* h, const float* xyzi_host, int n, int32_t id, int32_t* slot) {
  if (!h || !xyzi_host || n <= 0) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->ndt->stream;
  if (h->pool_n + (size_t)n > (size_t)INT32_MAX) { set_error("lsd_overlap_add_keyframe: key-frame pool above 2^31 points"); return LSD_ERR_CAPACITY; }
  if (h->pool_n + (size_t)n > h->pool_cap) {
    const size_t cap = std::max(h->pool_n + (size_t)n, 2 * h->pool_cap);
    float4* np_ = nullptr;
    LSD_CUDA(cudaMalloc((void**)&np_, cap * 16));
    if (h->pool_n) LSD_CUDA(cudaMemcpyAsync(np_, h->d_pool, h->pool_n * 16, cudaMemcpyDeviceToDevice, st));
    LSD_CUDA(cudaStreamSynchronize(st));
    cudaFree(h->d_pool);
    h->d_pool = np_; h->pool_cap = cap;
    // the filtered copies live in their own buffers; NDT tables and point maps hold copies of the points, not pointers
  }
  LSD_CUDA(cudaMemcpyAsync(h->d_pool + h->pool_n, xyzi_host, (size_t)n * 16, cudaMemcpyHostToDevice, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  if (slot) *slot = (int32_t)h->kf_n.size();
  h->kf_off.push_back(h->pool_n); h->kf_n.push_back(n); h->kf_id.push_back(id);
  h->tgt_of.push_back(-1);
  h->pool_n += (size_t)n;
  return LSD_OK;
}

lsd_status_t lsd_overlap_release_targets(lsd_overlap_t* h) {
  if (!h) return LSD_ERR_INVALID;
  ov_release_targets(h);
  return LSD_OK;
}

lsd_status_t lsd_overlap_find_candidates(const lsd_overlap_params_t* p, const double* poses16, const int32_t* ids, int n_slots,
                                         const int32_t* keyframes, int n_kf, const int32_t* edges, int n_e, int32_t new_slot,
                                         int32_t* cand_out, int cap, int* n_cand) {
  if (!p || !poses16 || !ids || n_slots < 0 || n_kf < 0 || n_e < 0 || (n_kf > 0 && !keyframes) || (n_e > 0 && !edges) || !n_cand ||
      (cap > 0 && !cand_out)) {
    set_error("lsd_overlap_find_candidates: bad arguments");
    return LSD_ERR_INVALID;
  }
  bool ok = new_slot >= 0 && new_slot < n_slots;
  for (int i = 0; ok && i < n_kf; i++) ok = keyframes[i] >= 0 && keyframes[i] < n_slots;
  if (!ok) { set_error("lsd_overlap_find_candidates: a slot outside [0, n_slots)"); return LSD_ERR_INVALID; }
  std::vector<int32_t> c;
  ov_find(*p, poses16, ids, keyframes, n_kf, ov_connections(edges, n_e), new_slot, c);
  *n_cand = (int)c.size();
  for (int i = 0; i < std::min(cap, *n_cand); i++) cand_out[i] = c[i];
  return LSD_OK;
}

void lsd_overlap_guess(const double* T_new16, const double* T_cand16, float* guess16) {
  if (T_new16 && T_cand16 && guess16) ov_guess(T_new16, T_cand16, guess16);
}

void lsd_overlap_finetune_guess(const float* ndt_final16, float* guess16) {
  if (ndt_final16 && guess16) ov_inverse_f(ndt_final16, guess16);
}

lsd_status_t lsd_overlap_fitness(lsd_overlap_t* h, int32_t target_slot, int32_t source_slot, const float* T16, double max_range,
                                 double* score, double* inlier_ratio, int* n_counted, int* n_filtered, int* target_incomplete) {
  if (!h || !T16 || !ov_slots_ok(h, &target_slot, 1) || !ov_slots_ok(h, &source_slot, 1)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(h->device));
  long long ln = 0;
  lsd_status_t s = ov_filtered_targets(h, std::vector<int>{target_slot}, &ln);
  if (s) return s;
  const lsd_overlap::Target& t = ov_target(h, target_slot);
  OvScreen q;
  q.src_slot = source_slot; q.tgt_pts = t.d_filt; q.tgt_n = t.n_filt; q.tgt_map = t.filt_map();
  memcpy(q.T, T16, sizeof(q.T));
  std::vector<double> sum, nr, nf;
  s = ov_prescreen(h, std::vector<OvScreen>{q}, max_range, sum, nr, nf, &ln);
  if (s) return s;
  double sc = 0, ratio = 0;
  ov_score(sum[0], nr[0], nf[0], &sc, &ratio);
  if (score) *score = sc;
  if (inlier_ratio) *inlier_ratio = ratio;
  if (n_counted) *n_counted = (int)nr[0];
  if (n_filtered) *n_filtered = (int)nf[0];
  if (target_incomplete) *target_incomplete = t.filt_map() ? (int)t.fmap->incomplete : 0;
  return LSD_OK;
}

lsd_status_t lsd_overlap_match(lsd_overlap_t* h, const int32_t* new_slots, const int32_t* cand_slots, const double* guesses16, int n,
                               int serial, double* final16, int32_t* converged, int32_t* iterations, double* fitness, long long* launches, int* rounds) {
  if (!h || n < 0 || (n > 0 && (!new_slots || !cand_slots || !guesses16)) || !ov_slots_ok(h, new_slots, n) || !ov_slots_ok(h, cand_slots, n)) {
    set_error("lsd_overlap_match: bad slots / arguments");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  long long ln = 0; int rd = 0;
  const std::vector<int> ns(new_slots, new_slots + n), cs(cand_slots, cand_slots + n);
  lsd_status_t s = serial ? ov_serial(h, ns, cs, guesses16, &ln, &rd) : ov_coarse(h, ns, cs, guesses16, &ln, &rd);
  if (s) return s;
  for (int i = 0; i < n; i++) {
    if (final16) memcpy(final16 + 16 * (size_t)i, h->lm[i].x0, 16 * sizeof(double));
    if (converged) converged[i] = h->lm[i].converged;
    if (iterations) iterations[i] = h->lm[i].iterations;
    if (fitness) fitness[i] = h->fitness[i];
  }
  if (launches) *launches = ln;
  if (rounds) *rounds = rd;
  return LSD_OK;
}

lsd_status_t lsd_overlap_iteration_log(lsd_overlap_t* h, int i, double* out4_per_iter, int cap_iters, int* n_iters) {
  if (!h || !n_iters || i < 0 || i >= (int)h->lm.size()) return LSD_ERR_INVALID;
  const std::vector<double>& lg = h->lm[i].iter_log;
  const int n = (int)(lg.size() / 4);
  *n_iters = n;
  if (out4_per_iter) memcpy(out4_per_iter, lg.data(), (size_t)std::min(n, std::max(cap_iters, 0)) * 4 * sizeof(double));
  return LSD_OK;
}

lsd_status_t lsd_overlap_last_reports(lsd_overlap_t* h, lsd_overlap_report_t* out, int cap, int* n) {
  if (!h || !n) return LSD_ERR_INVALID;
  *n = (int)h->reports.size();
  if (out) memcpy(out, h->reports.data(), (size_t)std::min(*n, std::max(cap, 0)) * sizeof(lsd_overlap_report_t));
  return LSD_OK;
}

lsd_status_t lsd_overlap_last_stats(lsd_overlap_t* h, long long* launches, int* rounds, int* target_buffers, int* targets_held) {
  if (!h) return LSD_ERR_INVALID;
  if (launches) *launches = h->last_launches;
  if (rounds) *rounds = h->last_rounds;
  if (target_buffers) *target_buffers = (int)h->targets.size();
  if (targets_held) *targets_held = (int)(h->targets.size() - h->free_targets.size());
  return LSD_OK;
}

// OverlapDetector::detect (:63-110) -> find_candidates (:113-145) -> matching (:147-211), every new key frame's prescreen
// and NDT batched together, the finetune one new key frame after another.
lsd_status_t lsd_overlap_detect(lsd_overlap_t* h, const double* poses16, const int32_t* keyframes, int n_kf, const int32_t* new_keyframes,
                                int n_new, const int32_t* edges, int n_e, lsd_overlap_result_t* out, int cap, int* n_found) {
  if (!h || !poses16 || !n_found || n_kf < 0 || n_new < 0 || n_e < 0 || (n_kf > 0 && !keyframes) || (n_new > 0 && !new_keyframes) ||
      (n_e > 0 && !edges) || (cap > 0 && !out) || !ov_slots_ok(h, keyframes, n_kf) || !ov_slots_ok(h, new_keyframes, n_new)) {
    set_error("lsd_overlap_detect: bad slots / arguments");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  struct Release { lsd_overlap* h; ~Release() { ov_release_targets(h); } } release{h};   // tables scoped to the call
  *n_found = 0;
  h->reports.clear();
  long long ln = 0; int rd = 0;
  const ConnMap conn = ov_connections(edges, n_e);
  std::map<int, int> id_index;                                   // keyframe_id_map (:93-97)
  for (int i = 0; i < n_kf; i++) id_index[h->kf_id[keyframes[i]]] = i;
  // candidates and guesses of every new key frame
  std::vector<std::vector<int32_t>> cands(n_new);
  std::vector<OvScreen> screens;
  std::vector<int> screen_q;
  std::vector<int> targets;
  for (int q = 0; q < n_new; q++) {
    const int32_t ns = new_keyframes[q];
    ov_find(h->p, poses16, h->kf_id.data(), keyframes, n_kf, conn, ns, cands[q]);
    if (!cands[q].empty()) targets.push_back(ns);
    for (int32_t k : cands[q]) {
      OvScreen e;
      e.src_slot = k;
      ov_guess(poses16 + 16 * (size_t)ns, poses16 + 16 * (size_t)k, e.T);
      screens.push_back(e);
      screen_q.push_back(q);
    }
  }
  // prescreen (:160-163) of every pair: calc_fitness_score(new, candidate, guess, 1.0)
  lsd_status_t s = ov_filtered_targets(h, targets, &ln);
  if (s) return s;
  for (size_t i = 0; i < screens.size(); i++) {
    const lsd_overlap::Target& t = ov_target(h, new_keyframes[screen_q[i]]);
    screens[i].tgt_pts = t.d_filt; screens[i].tgt_n = t.n_filt; screens[i].tgt_map = t.filt_map();
  }
  std::vector<double> sum, nr, nf;
  s = ov_prescreen(h, screens, h->p.inlier_max_range, sum, nr, nf, &ln);
  if (s) return s;
  // NDT (:165-171) of every pair that passed, all new key frames together
  std::vector<int> pn, pc, pidx;
  std::vector<double> guesses;
  for (size_t i = 0; i < screens.size(); i++) {
    double sc = 0, ratio = 0;
    ov_score(sum[i], nr[i], nf[i], &sc, &ratio);
    if (ratio < h->p.fitness_inlier_thresh) continue;
    pn.push_back(new_keyframes[screen_q[i]]); pc.push_back(screens[i].src_slot); pidx.push_back((int)i);
    for (int e = 0; e < 16; e++) guesses.push_back((double)screens[i].T[e]);
  }
  s = ov_coarse(h, pn, pc, guesses.data(), &ln, &rd);
  if (s) return s;
  // per new key frame: the best candidate (:168-183), then the finetune (:185-210)
  size_t at = 0, pa = 0;
  for (int q = 0; q < n_new; q++) {
    const int32_t ns = new_keyframes[q];
    lsd_overlap_report_t rep;
    memset(&rep, 0, sizeof(rep));
    rep.new_slot = ns; rep.n_candidates = (int)cands[q].size(); rep.best_slot = -1; rep.best_score = DBL_MAX;
    int best = -1;
    double best_score = DBL_MAX;
    for (size_t j = 0; j < cands[q].size(); j++, at++) {
      if (pa < pidx.size() && pidx[pa] == (int)at) {
        rep.n_prescreened++;
        const int i = (int)pa++;
        if (!h->lm[i].converged) continue;
        if (h->fitness[i] > best_score) continue;   // an equal score replaces the previous best
        best_score = h->fitness[i];
        best = i;
      }
    }
    if (cands[q].empty()) { rep.decision = LSD_OVERLAP_NO_CANDIDATES; h->reports.push_back(rep); continue; }
    if (best < 0) { rep.decision = LSD_OVERLAP_NO_MATCH; h->reports.push_back(rep); continue; }
    rep.best_slot = pc[best]; rep.best_score = best_score;
    // finetune: target = best accumulated with its connected frames, source = the new key frame
    s = ov_accumulate(h, poses16, keyframes, n_kf, id_index, conn, pc[best], &ln);
    if (s) return s;
    rep.n_accum = h->n_accum;
    lsd_reg* g = h->gicp;
    const long long g0 = g->launches;
    s = lsd_reg_set_target_dev(g, reinterpret_cast<const float*>(h->d_accum), h->n_accum);
    if (!s) s = lsd_reg_set_source_dev(g, reinterpret_cast<const float*>(h->d_pool + h->kf_off[ns]), h->kf_n[ns]);
    if (s) return s;
    float ndt_f[16], gf[16];
    for (int e = 0; e < 16; e++) ndt_f[e] = (float)h->lm[best].x0[e];
    ov_inverse_f(ndt_f, gf);
    double gs[16];
    for (int e = 0; e < 16; e++) gs[e] = (double)gf[e];
    s = reg_align(g, gs);
    ln += g->launches - g0;
    if (s < 0) return s;
    if (!g->converged) { rep.decision = LSD_OVERLAP_GICP_DIVERGED; h->reports.push_back(rep); continue; }
    float Tf[16];
    for (int e = 0; e < 16; e++) Tf[e] = (float)g->final_T[e];
    // calc_fitness_score(accum, new, relative_pose, fitness_score_max_range) (:204): the accumulated target filtered
    s = grow_dev(h->d_accf, h->accf_cap, (size_t)h->n_accum);
    if (s) return s;
    std::vector<int> cnt;
    s = ov_filter(h, std::vector<OvFilt>{OvFilt{h->d_accum, h->d_accf, h->n_accum}}, cnt, &ln);
    if (s) return s;
    h->n_accf = cnt[0];
    s = ov_point_map(h, &h->accf_map, h->d_accf, h->n_accf, &ln);
    if (s) return s;
    OvScreen e;
    e.src_slot = ns; e.tgt_pts = h->d_accf; e.tgt_n = h->n_accf; e.tgt_map = h->n_accf > 0 ? h->accf_map : nullptr;
    memcpy(e.T, Tf, sizeof(Tf));
    std::vector<double> fs, fr, ff;
    s = ov_prescreen(h, std::vector<OvScreen>{e}, h->p.fitness_score_max_range, fs, fr, ff, &ln);
    if (s) return s;
    double score = 0, ratio = 0;
    ov_score(fs[0], fr[0], ff[0], &score, &ratio);
    rep.accum_incomplete = e.tgt_map ? (int)e.tgt_map->incomplete : 0;
    if (score > h->p.fitness_score_thresh) { rep.decision = LSD_OVERLAP_GICP_REJECT; rep.score = score; h->reports.push_back(rep); continue; }
    rep.decision = LSD_OVERLAP_FOUND;
    rep.score = score;
    h->reports.push_back(rep);
    if (*n_found < cap) {
      lsd_overlap_result_t& r = out[*n_found];
      memset(&r, 0, sizeof(r));
      r.key1 = pc[best]; r.key2 = ns;
      for (int k = 0; k < 16; k++) r.relpose16[k] = (double)Tf[k];   // relative_pose.cast<double>() (:210)
      r.score = score; r.coarse_score = best_score;
    }
    (*n_found)++;
  }
  h->last_launches = ln; h->last_rounds = rd;
  return LSD_OK;
}

}  // extern "C"
