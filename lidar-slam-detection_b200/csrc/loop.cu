// loop.cu — loop-closure detector: hdl_graph_slam::LoopDetector (loop_detector.hpp:33-231) with its coarse stage batched
// over the candidate set, and the fitness of InformationMatrixCalculator (information_matrix_calculator.cpp:25-47,71-102).
//
// The reference aligns the candidates one after another (:158-191), each with NDT_CUDA's Levenberg-Marquardt loop: one
// cost evaluation, one host round trip.  Here every candidate keeps its own LM state (LmState, reg.cu) and the states
// advance together: one ndt_cost_batch_kernel launch per round evaluates the next cost of every live candidate against
// the new key frame's NDT map, so a detect costs as many round trips as its slowest candidate, not their sum.
// Per candidate the launch is the single-pair launch: reg_grid(n_c) blocks with the same point-to-block partition, the
// per-point body ndt_cost_kernel runs (ndt_point, reg.cu), the same block_partials<29> and a last-block fold over those
// blocks in grid_finalize's order — H, b, err and the correspondence count are the bits of ndt_cost_kernel, so the LM
// trajectory is that of a separate lsd_reg handle.  The fitness launch runs lsd_reg_fitness's body (fitness_range).
// Included by lsdreg.cu after reg.cu (uses its kernels' building blocks and the host helpers).

namespace lsd {

// One candidate of a batched launch: where its blocks, points and correspondences are.
struct LoopCand {
  int src_off, n;        // first point in the key-frame pool, point count
  int blk_off, n_blk;    // first block of the launch, blocks it gets (the single-pair grid for n)
  long long corr_off;    // NDT: [n_off, n] correspondence slots at this offset of the correspondence pool
  int row;               // result row (candidate index in the caller's list)
  int update, deriv;     // NDT: linearize (refresh correspondences) / accumulate H and b
  int warp_shape;        // fitness: fitness_range<true> (one warp per point) instead of <false> (one thread), as lsd_reg_fitness
  Pose34f lin, ev;       // NDT: linearisation / evaluation pose; fitness: ev is the pose
};

// The candidate a block belongs to (blk_off ascending): computed once per block.  Cand: LoopCand here, GaCand in galign.cu.
template <class Cand>
__device__ __forceinline__ int loop_cand_of_block(const Cand* __restrict__ cands, int n_cand) {
  __shared__ int s_c;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n_cand - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (cands[mid].blk_off <= (int)blockIdx.x) lo = mid; else hi = mid - 1; }
    s_c = lo;
  }
  __syncthreads();
  return s_c;
}

// grid_finalize (lio.cu) for the G blocks of one candidate: the last of them folds partials[0 .. G) in the same order
// (slices of blocks, ascending, then the slices) into its result row.  The last candidate to finish publishes `seq` —
// one publication per launch, which the host spins on (wait_seq).
template <int NV>
__device__ __forceinline__ void loop_finalize(const double* __restrict__ partials, int G, unsigned* __restrict__ done_c,
                                              unsigned* __restrict__ done_all, int n_cand, volatile double* __restrict__ row,
                                              volatile double* __restrict__ seq_slot, double seq) {
  __shared__ double sm_fin[8][kNV];
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(done_c, 1u) == (unsigned)G - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int slices = blockDim.x >> 5;
  const int j = threadIdx.x & 31, slice = threadIdx.x >> 5;
  double s = 0.0;
  if (j < NV) {
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
    row[threadIdx.x] = t;
  }
  if (threadIdx.x == NV) *done_c = 0u;
  if (threadIdx.x <= NV) __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(done_all, 1u) == (unsigned)n_cand - 1) {
    __threadfence_system();
    *done_all = 0u;
    *seq_slot = seq;  // published last
  }
}

// One cost evaluation for every candidate of the launch, all against the new key frame's NDT map.
__global__ void __launch_bounds__(256) ndt_cost_batch_kernel(NdtView v, const float4* __restrict__ pool, const LoopCand* __restrict__ cands,
                                                             int n_cand, int n_off, int* __restrict__ corr_pool, double* __restrict__ partials,
                                                             unsigned* __restrict__ done, double* __restrict__ result, double seq) {
  const int c = loop_cand_of_block(cands, n_cand);
  const int n = cands[c].n, G = cands[c].n_blk, lb = (int)blockIdx.x - cands[c].blk_off;
  const bool update = cands[c].update != 0, deriv = cands[c].deriv != 0;
  const Pose34f lin = cands[c].lin, ev = cands[c].ev;
  const float4* src = pool + cands[c].src_off;
  int* corr = corr_pool + cands[c].corr_off;
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = lb * blockDim.x + threadIdx.x; i < n; i += G * blockDim.x)
    ndt_point(v, __ldg(src + i), i, n, n_off, lin, ev, corr, update, deriv, vals);
  block_partials<29>(vals, partials);  // row blockIdx.x = blk_off + lb
  loop_finalize<29>(partials + (size_t)cands[c].blk_off * kNV, G, done + 1 + c, done, n_cand,
                    result + (size_t)(1 + cands[c].row) * kNV, result, seq);
}

// getFitnessScore(max_range) of every candidate at its pose against the new key frame's point map.  Per candidate the
// shape and grid of lsd_reg_fitness and the same body (fitness_range, reg.cu) and fold: same sum, same count.
// tg: the new key frame's cloud as the fallback of the map's grid search (fitness_target).
__global__ void __launch_bounds__(kRegWarps * 32, 2) fitness_batch_kernel(MapView mv, const float4* __restrict__ pool,
                                                                          const LoopCand* __restrict__ cands, int n_cand, float search_sq,
                                                                          double max_range, NnTarget tg,
                                                                          double* __restrict__ partials, unsigned* __restrict__ done,
                                                                          double* __restrict__ result, double seq) {
  const int c = loop_cand_of_block(cands, n_cand);
  const int n = cands[c].n, G = cands[c].n_blk, lb = (int)blockIdx.x - cands[c].blk_off;
  const Pose34f Tf = cands[c].ev;
  const float4* src = pool + cands[c].src_off;
  if (cands[c].warp_shape)  // block-uniform
    fitness_range<true>(mv, src, n, lb, G, Tf, search_sq, max_range, tg, partials);
  else
    fitness_range<false>(mv, src, n, lb, G, Tf, search_sq, max_range, tg, partials);
  loop_finalize<2>(partials + (size_t)cands[c].blk_off * kNV, G, done + 1 + c, done, n_cand,
                   result + (size_t)(1 + cands[c].row) * kNV, result, seq);
}

}  // namespace lsd

// ==================================================================== host side
namespace lsd {

// Host side of a batched launch (the loop detector's candidates here, the global aligner's pairs in galign.cu): the
// descriptors, partial rows, per-candidate done counters and mapped result rows, grown to the largest batch seen so that a
// round allocates nothing.  Result row 0 holds the sequence number the last candidate to finish publishes (loop_finalize),
// row 1 + c the sums of candidate c.
template <class Cand>
struct BatchScratch {
  Cand* d_cand = nullptr; Cand* h_cand = nullptr; int cand_cap = 0;
  double* d_partials = nullptr; size_t part_cap = 0;     // rows of kNV doubles
  unsigned* d_done = nullptr;                            // [0] candidates finished, [1 + c] blocks of candidate c finished; self-resetting
  double *h_res = nullptr, *d_res = nullptr;             // mapped
  long long seq = 0;

  // room for n candidates and `rows` partial rows
  lsd_status_t reserve(int n, size_t rows) {
    if (n > cand_cap) {
      cudaFree(d_cand); cudaFreeHost(h_cand); cudaFree(d_done); cudaFreeHost(h_res);
      d_cand = nullptr; h_cand = nullptr; d_done = nullptr; h_res = nullptr; cand_cap = 0;
      const int cap = std::max(n, 32);
      LSD_CUDA(cudaMalloc((void**)&d_cand, cap * sizeof(Cand)));
      LSD_CUDA(cudaHostAlloc((void**)&h_cand, cap * sizeof(Cand), cudaHostAllocDefault));
      LSD_CUDA(cudaMalloc((void**)&d_done, (cap + 1) * sizeof(unsigned)));
      LSD_CUDA(cudaMemset(d_done, 0, (cap + 1) * sizeof(unsigned)));
      LSD_CUDA(cudaHostAlloc((void**)&h_res, (size_t)(cap + 1) * kNV * 8, cudaHostAllocMapped));
      memset(h_res, 0, (size_t)(cap + 1) * kNV * 8);
      LSD_CUDA(cudaHostGetDevicePointer((void**)&d_res, h_res, 0));
      cand_cap = cap;
    }
    if (rows > part_cap) {
      cudaFree(d_partials); d_partials = nullptr; part_cap = 0;
      LSD_CUDA(cudaMalloc((void**)&d_partials, rows * kNV * 8));
      part_cap = rows;
    }
    return LSD_OK;
  }
  // h_cand[0, n) to the device on st; *s = the sequence number the launch is to publish
  lsd_status_t upload(int n, cudaStream_t st, double* s) {
    LSD_CUDA(cudaMemcpyAsync(d_cand, h_cand, n * sizeof(Cand), cudaMemcpyHostToDevice, st));
    *s = (double)(++seq);
    return LSD_OK;
  }
  lsd_status_t wait(cudaStream_t st, double s) const { return wait_seq(h_res, st, s, 20.0); }
  const double* row(int i) const { return h_res + (size_t)(1 + i) * kNV; }
  void release() { cudaFree(d_cand); cudaFreeHost(h_cand); cudaFree(d_partials); cudaFree(d_done); cudaFreeHost(h_res); }
};

// A device buffer of at least n elements (contents not kept); true in *grown when it was reallocated.
template <class T>
static lsd_status_t grow_dev(T*& p, size_t& cap, size_t n, bool* grown = nullptr) {
  if (grown) *grown = n > cap;
  if (n <= cap) return LSD_OK;
  cudaFree(p); p = nullptr; cap = 0;
  LSD_CUDA(cudaMalloc((void**)&p, n * sizeof(T)));
  cap = n;
  return LSD_OK;
}

}  // namespace lsd

struct lsd_loop {
  lsd_loop_params_t p{};
  int device = 0;
  lsd_reg* ndt = nullptr;    // coarse stage: owns the stream, the new key frame's NDT map and its point map (fitness)
  lsd_reg* gicp = nullptr;   // refinement (FAST_GICP, max-corr 0.5 m)
  int target_slot = -1;      // key frame whose maps `ndt` holds
  // key-frame pool: every cloud once, [sum n, 4] float
  float4* d_pool = nullptr; size_t pool_n = 0, pool_cap = 0;
  std::vector<size_t> kf_off;
  std::vector<int> kf_n;
  std::vector<double> kf_accum;
  double last_edge = 0.0;    // last_edge_accum_distance (loop_detector.hpp:60,216)
  // batch scratch, grown to the largest candidate set seen
  lsd::BatchScratch<lsd::LoopCand> b;
  int* d_corr = nullptr; size_t corr_cap = 0;
  // last lsd_loop_match
  std::vector<lsd::LmState> lm;
  std::vector<double> fitness;
  std::vector<lsd_loop_report_t> reports;
};

namespace lsd {

static lsd_status_t loop_reserve(lsd_loop* h, const std::vector<int>& ns, int n_off) {
  size_t rows = 0, corr = 0;
  for (int v : ns) { rows += (size_t)std::max(reg_grid(v), warp_grid(v)); corr += (size_t)n_off * v; }
  lsd_status_t s = h->b.reserve((int)ns.size(), rows);
  if (s) return s;
  return grow_dev(h->d_corr, h->corr_cap, corr);
}

// setInputTarget(new_keyframe->cloud) (:156): NDT map of the target, plus its exact-NN point map for the fitness scores.
static lsd_status_t loop_set_target(lsd_loop* h, int slot, long long* launches) {
  if (h->target_slot == slot) return LSD_OK;
  h->target_slot = -1;
  lsd_reg* r = h->ndt;
  const long long l0 = r->launches;
  lsd_status_t s = lsd_reg_set_target_dev(r, reinterpret_cast<const float*>(h->d_pool + h->kf_off[slot]), h->kf_n[slot]);
  if (s) return s;
  s = build_point_map(r, &r->tgt_map, r->d_tgt, r->n_tgt);
  if (s) return s;
  r->launches++;
  r->tgt_map_built = true;
  *launches += r->launches - l0;
  h->target_slot = slot;
  return LSD_OK;
}

// One fitness launch for candidates (slot, pose) against the current target; score[i] as getFitnessScore returns it.
static lsd_status_t loop_fitness(lsd_loop* h, const std::vector<int>& slots, const std::vector<Pose34f>& poses, double max_range,
                                 double* score, double* count, long long* launches) {
  const int n = (int)slots.size();
  if (n == 0) return LSD_OK;
  lsd_reg* r = h->ndt;
  std::vector<int> ns(n);
  for (int i = 0; i < n; i++) ns[i] = h->kf_n[slots[i]];
  lsd_status_t s = loop_reserve(h, ns, r->p.ndt_neighbors);
  if (s) return s;
  int blocks = 0;
  for (int i = 0; i < n; i++) {
    LoopCand& c = h->b.h_cand[i];
    memset(&c, 0, sizeof(c));
    c.src_off = (int)h->kf_off[slots[i]]; c.n = ns[i]; c.row = i;
    c.warp_shape = ns[i] < kThreadShapeMin;
    c.n_blk = c.warp_shape ? warp_grid(ns[i]) : reg_grid(ns[i]);
    c.blk_off = blocks; blocks += c.n_blk;
    c.ev = poses[i]; c.lin = poses[i];
  }
  cudaStream_t st = r->stream;
  double seq = 0;
  s = h->b.upload(n, st, &seq);
  if (s) return s;
  const float search_sq = fitness_search_sq(max_range, r->p.map_resolution);
  fitness_batch_kernel<<<blocks, kRegWarps * 32, 0, st>>>(r->tgt_map->view, h->d_pool, h->b.d_cand, n, search_sq, max_range,
                                                         fitness_target(r->tgt_map, r->d_tgt, r->n_tgt, max_range, r->p.map_resolution),
                                                         h->b.d_partials, h->b.d_done, h->b.d_res, seq);
  LSD_CUDA(cudaGetLastError());
  (*launches)++;
  s = h->b.wait(st, seq);
  if (s) return s;
  for (int i = 0; i < n; i++) {
    const double sum = h->b.row(i)[0], cnt = h->b.row(i)[1];
    score[i] = cnt > 0 ? sum / cnt : DBL_MAX;
    if (count) count[i] = cnt;
  }
  return LSD_OK;
}

// The coarse stage for candidates `cand` (guesses in double) against key frame `target`: every candidate's LM loop of
// lsd_reg_align, advanced together, then getFitnessScore(fitness_score_max_range) of all of them in one launch.
static lsd_status_t loop_coarse(lsd_loop* h, int target, const int32_t* cand, const double* guesses, int n, long long* launches, int* rounds) {
  *launches = 0; *rounds = 0;
  lsd_status_t s = loop_set_target(h, target, launches);
  if (s) return s;
  lsd_reg* r = h->ndt;
  const int n_off = r->p.ndt_neighbors;
  std::vector<int> ns(n);
  for (int i = 0; i < n; i++) ns[i] = h->kf_n[cand[i]];
  s = loop_reserve(h, ns, n_off);
  if (s) return s;
  std::vector<long long> corr_off(n);
  long long co = 0;
  for (int i = 0; i < n; i++) { corr_off[i] = co; co += (long long)n_off * ns[i]; }
  h->lm.assign(n, LmState());
  for (int i = 0; i < n; i++) lm_begin(h->lm[i], h->p.coarse, guesses + 16 * (size_t)i);
  cudaStream_t st = r->stream;
  for (;;) {
    int na = 0, blocks = 0;
    for (int i = 0; i < n; i++) {
      const LmState& m = h->lm[i];
      if (m.done) continue;
      LoopCand& c = h->b.h_cand[na++];
      memset(&c, 0, sizeof(c));
      c.src_off = (int)h->kf_off[cand[i]]; c.n = ns[i]; c.row = i;
      c.n_blk = reg_grid(ns[i]); c.blk_off = blocks; blocks += c.n_blk;
      c.corr_off = corr_off[i];
      c.update = m.want_update; c.deriv = m.want_update;
      T_to_pose(m.want_T, nullptr, &c.ev);
      c.lin = c.ev;   // read only when update (the linearisation pose is the evaluation pose then)
    }
    if (na == 0) break;
    double seq = 0;
    s = h->b.upload(na, st, &seq);
    if (s) return s;
    ndt_cost_batch_kernel<<<blocks, 256, 0, st>>>(r->ndt, h->d_pool, h->b.d_cand, na, n_off, h->d_corr, h->b.d_partials, h->b.d_done,
                                                  h->b.d_res, seq);
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
  std::vector<int> slots(cand, cand + n);
  std::vector<Pose34f> poses(n);
  for (int i = 0; i < n; i++) T_to_pose(h->lm[i].x0, nullptr, &poses[i]);
  h->fitness.assign(n, 0.0);
  return loop_fitness(h, slots, poses, h->p.fitness_score_max_range, h->fitness.data(), nullptr, launches);
}

// Eigen::Quaterniond(R).normalized().toRotationMatrix() (Eigen/src/Geometry/Quaternion.h quaternionbase_assign_impl,
// toRotationMatrix), R row-major 3x3 taken from a 4x4
static void normalize_rotation(const double* T, double* R) {
  auto m = [&](int i, int j) { return T[4 * i + j]; };
  double q[4];  // x y z w
  const double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0) {
    double s = sqrt(t + 1.0);
    q[3] = 0.5 * s; s = 0.5 / s;
    q[0] = (m(2, 1) - m(1, 2)) * s; q[1] = (m(0, 2) - m(2, 0)) * s; q[2] = (m(1, 0) - m(0, 1)) * s;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
    q[i] = 0.5 * s; s = 0.5 / s;
    q[3] = (m(k, j) - m(j, k)) * s; q[j] = (m(j, i) + m(i, j)) * s; q[k] = (m(k, i) + m(i, k)) * s;
  }
  const double nrm = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (double& v : q) v /= nrm;
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x,
               tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

// guess of :165-173: (new^-1 * candidate) in double, cast to float, (2,3) zeroed
static void loop_guess(const double* Tnew, const double* Tcand, double* G) {
  double Rn[9], Rc[9];
  normalize_rotation(Tnew, Rn);
  normalize_rotation(Tcand, Rc);
  const double tn[3] = {Tnew[3], Tnew[7], Tnew[11]}, tc[3] = {Tcand[3], Tcand[7], Tcand[11]};
  double Ri[9], ti[3];  // Isometry inverse: R^T, -R^T t
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) Ri[3 * a + b] = Rn[3 * b + a];
  for (int a = 0; a < 3; a++) ti[a] = -(Ri[3 * a] * tn[0] + Ri[3 * a + 1] * tn[1] + Ri[3 * a + 2] * tn[2]);
  for (int i = 0; i < 16; i++) G[i] = 0.0;
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) G[4 * a + b] = Ri[3 * a] * Rc[b] + Ri[3 * a + 1] * Rc[3 + b] + Ri[3 * a + 2] * Rc[6 + b];
    G[4 * a + 3] = (Ri[3 * a] * tc[0] + Ri[3 * a + 1] * tc[1] + Ri[3 * a + 2] * tc[2]) + ti[a];
  }
  G[15] = 1.0;
  for (int i = 0; i < 16; i++) G[i] = (double)(float)G[i];
  G[11] = 0.0;
}

// find_candidates (:106-140)
static int loop_find(const lsd_loop_params_t& p, double last_edge, const double* poses16, const double* accum, const int32_t* kfs, int n_kf,
                     int32_t ns, std::vector<int32_t>& out) {
  out.clear();
  if (accum[ns] - last_edge < p.distance_from_last_edge_thresh) return 0;
  double acc_kf = -100.0;
  const double* Tn = poses16 + 16 * (size_t)ns;
  for (int i = 0; i < n_kf; i++) {
    const int32_t k = kfs[i];
    if (accum[ns] - accum[k] < p.accum_distance_thresh) continue;
    if (accum[k] - acc_kf < p.distance_keyframe_thresh) continue;
    const double* Tk = poses16 + 16 * (size_t)k;
    const double dx = Tk[3] - Tn[3], dy = Tk[7] - Tn[7];
    if (sqrt(dx * dx + dy * dy) > p.distance_thresh) continue;
    acc_kf = accum[k];
    out.push_back(k);
  }
  return (int)out.size();
}

// InformationMatrixCalculator (information_matrix_calculator.cpp:10-21 defaults, weight() in the header :44-47)
static void loop_information(double fitness, double* inf) {
  const double a = 20.0, thresh = 0.5;
  auto weight = [&](double min_y, double max_y) {
    const double y = (1.0 - exp(-a * fitness)) / (1.0 - exp(-a * thresh));
    return min_y + (max_y - min_y) * y;
  };
  const float w_x = (float)weight(pow(0.1, 2), pow(5.0, 2));
  const float w_q = (float)weight(pow(0.05, 2), pow(0.2, 2));
  for (int i = 0; i < 36; i++) inf[i] = (i % 7 == 0) ? 1.0 : 0.0;
  for (int i = 0; i < 3; i++) inf[7 * i] /= w_x;
  for (int i = 3; i < 6; i++) inf[7 * i] /= w_q;
}

}  // namespace lsd

using namespace lsd;

extern "C" {

void lsd_loop_default_params(lsd_loop_params_t* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->distance_thresh = 15.0;                 // loop_detector.hpp:43-50
  p->accum_distance_thresh = 25.0;
  p->distance_from_last_edge_thresh = 15.0;
  p->distance_new_keyframe_thresh = 2.0;
  p->distance_keyframe_thresh = 2.0;
  p->fitness_score_max_range = 25.0;
  p->fitness_score_thresh = 1.5;
  lsd_reg_default_params(&p->coarse, LSD_REG_NDT_P2D);   // select_registration_method("NDT_CUDA") (:53)
  lsd_reg_default_params(&p->accurate, LSD_REG_GICP);    // select_registration_method("FAST_GICP") (:57-59)
  p->accurate.max_corr_dist = 0.5;
}

lsd_status_t lsd_loop_create(lsd_loop_t** out, const lsd_loop_params_t* p) {
  if (!out || !p) return LSD_ERR_INVALID;
  if (p->coarse.kind != LSD_REG_NDT_P2D || p->accurate.kind == LSD_REG_NDT_P2D) {
    set_error("lsd_loop_create: the coarse stage is NDT_P2D, the refinement GICP or VGICP");
    return LSD_ERR_INVALID;
  }
  if (p->coarse.max_process_time_us != 0) { set_error("lsd_loop_create: the coarse stage has no timeout (loop_detector.hpp:53)"); return LSD_ERR_INVALID; }
  lsd_loop* h = new lsd_loop();
  h->p = *p;
  lsd_status_t s = lsd_reg_create(&h->ndt, &p->coarse);
  if (!s) s = lsd_reg_create(&h->gicp, &p->accurate);
  if (s) { lsd_loop_destroy(h); return s; }
  h->device = h->ndt->device;
  *out = h;
  return LSD_OK;
}

lsd_status_t lsd_loop_destroy(lsd_loop_t* h) {
  if (!h) return LSD_OK;
  if (h->ndt) { cudaSetDevice(h->ndt->device); cudaStreamSynchronize(h->ndt->stream); }
  cudaFree(h->d_pool); cudaFree(h->d_corr);
  h->b.release();
  lsd_reg_destroy(h->ndt);
  lsd_reg_destroy(h->gicp);
  delete h;
  return LSD_OK;
}

lsd_status_t lsd_loop_add_keyframe(lsd_loop_t* h, const float* xyzi_host, int n, double accum_distance, int32_t* slot) {
  if (!h || !xyzi_host || n <= 0) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->ndt->stream;
  if (h->pool_n + (size_t)n > (size_t)INT32_MAX) { set_error("lsd_loop_add_keyframe: key-frame pool above 2^31 points"); return LSD_ERR_CAPACITY; }
  if (h->pool_n + (size_t)n > h->pool_cap) {
    const size_t cap = std::max(h->pool_n + (size_t)n, 2 * h->pool_cap);
    float4* np_ = nullptr;
    LSD_CUDA(cudaMalloc((void**)&np_, cap * 16));
    if (h->pool_n) LSD_CUDA(cudaMemcpyAsync(np_, h->d_pool, h->pool_n * 16, cudaMemcpyDeviceToDevice, st));
    LSD_CUDA(cudaStreamSynchronize(st));
    cudaFree(h->d_pool);
    h->d_pool = np_; h->pool_cap = cap;
  }
  LSD_CUDA(cudaMemcpyAsync(h->d_pool + h->pool_n, xyzi_host, (size_t)n * 16, cudaMemcpyHostToDevice, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  if (slot) *slot = (int32_t)h->kf_n.size();
  h->kf_off.push_back(h->pool_n); h->kf_n.push_back(n); h->kf_accum.push_back(accum_distance);
  h->pool_n += (size_t)n;
  return LSD_OK;
}

lsd_status_t lsd_loop_find_candidates(const lsd_loop_params_t* p, double last_edge_accum_distance, const double* poses16,
                                      const double* accum, const int32_t* keyframes, int n_kf, int32_t new_slot,
                                      int32_t* cand_out, double* guesses16_out, int cap, int* n_cand) {
  if (!p || !poses16 || !accum || (n_kf > 0 && !keyframes) || new_slot < 0 || !n_cand || (cap > 0 && !cand_out)) return LSD_ERR_INVALID;
  std::vector<int32_t> c;
  *n_cand = loop_find(*p, last_edge_accum_distance, poses16, accum, keyframes, n_kf, new_slot, c);
  for (int i = 0; i < std::min(cap, *n_cand); i++) {
    cand_out[i] = c[i];
    if (guesses16_out) loop_guess(poses16 + 16 * (size_t)new_slot, poses16 + 16 * (size_t)c[i], guesses16_out + 16 * (size_t)i);
  }
  return LSD_OK;
}

static bool slots_ok(const lsd_loop* h, const int32_t* s, int n) {
  for (int i = 0; i < n; i++) if (s[i] < 0 || s[i] >= (int32_t)h->kf_n.size()) return false;
  return true;
}

lsd_status_t lsd_loop_match(lsd_loop_t* h, int32_t target_slot, const int32_t* cand, const double* guesses16, int n,
                            double* final16, int32_t* converged, int32_t* iterations, double* fitness, long long* launches,
                            int* rounds) {
  if (!h || n < 0 || (n > 0 && (!cand || !guesses16)) || !slots_ok(h, &target_slot, 1) || !slots_ok(h, cand, n)) {
    set_error("lsd_loop_match: bad slots / arguments");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  long long ln = 0; int rd = 0;
  lsd_status_t s = n > 0 ? loop_coarse(h, target_slot, cand, guesses16, n, &ln, &rd) : LSD_OK;
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

lsd_status_t lsd_loop_iteration_log(lsd_loop_t* h, int i, double* out4_per_iter, int cap_iters, int* n_iters) {
  if (!h || !n_iters || i < 0 || i >= (int)h->lm.size()) return LSD_ERR_INVALID;
  const std::vector<double>& lg = h->lm[i].iter_log;
  const int n = (int)(lg.size() / 4);
  *n_iters = n;
  if (out4_per_iter) memcpy(out4_per_iter, lg.data(), (size_t)std::min(n, std::max(cap_iters, 0)) * 4 * sizeof(double));
  return LSD_OK;
}

lsd_status_t lsd_loop_fitness(lsd_loop_t* h, int32_t target_slot, int32_t source_slot, const float* T16, double max_range,
                              double* score, int* n_counted) {
  if (!h || !T16 || !score || !slots_ok(h, &target_slot, 1) || !slots_ok(h, &source_slot, 1)) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(h->device));
  long long ln = 0;
  lsd_status_t s = loop_set_target(h, target_slot, &ln);
  if (s) return s;
  double T[16];
  for (int i = 0; i < 16; i++) T[i] = (double)T16[i];
  std::vector<Pose34f> pose(1);
  T_to_pose(T, nullptr, &pose[0]);
  double cnt = 0;
  s = loop_fitness(h, std::vector<int>{source_slot}, pose, max_range, score, &cnt, &ln);
  if (n_counted) *n_counted = (int)(cnt + 0.5);
  return s;
}

void lsd_loop_information_matrix(double fitness_score, double* information36) {
  if (information36) loop_information(fitness_score, information36);
}

lsd_status_t lsd_loop_last_edge(lsd_loop_t* h, double* value, int get) {
  if (!h || !value) return LSD_ERR_INVALID;
  if (get) *value = h->last_edge; else h->last_edge = *value;
  return LSD_OK;
}

lsd_status_t lsd_loop_last_reports(lsd_loop_t* h, lsd_loop_report_t* out, int cap, int* n) {
  if (!h || !n) return LSD_ERR_INVALID;
  *n = (int)h->reports.size();
  if (out) memcpy(out, h->reports.data(), (size_t)std::min(*n, std::max(cap, 0)) * sizeof(lsd_loop_report_t));
  return LSD_OK;
}

// LoopDetector::detect (:69-91) -> find_candidates (:106-140) -> matching (:148-219), and the information matrix the caller
// computes for the edge (hdl_graph_slam_nodelet.cpp:613-620, information_matrix_calculator.cpp:25-47).
lsd_status_t lsd_loop_detect(lsd_loop_t* h, const double* poses16, const int32_t* keyframes, int n_kf,
                             const int32_t* new_keyframes, int n_new, lsd_loop_result_t* out, int cap, int* n_loops) {
  if (!h || !poses16 || !n_loops || n_kf < 0 || n_new < 0 || (n_kf > 0 && !keyframes) || (n_new > 0 && !new_keyframes) ||
      (cap > 0 && !out) || !slots_ok(h, keyframes, n_kf) || !slots_ok(h, new_keyframes, n_new)) {
    set_error("lsd_loop_detect: bad slots / arguments");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  *n_loops = 0;
  h->reports.clear();
  const double* accum = h->kf_accum.data();
  double acc_new = 0.0;   // accum_distance_new_keyframe (:73)
  std::vector<int32_t> cand;
  std::vector<double> guesses;
  for (int q = 0; q < n_new; q++) {
    const int32_t ns = new_keyframes[q];
    lsd_loop_report_t rep = {ns, LSD_LOOP_SKIPPED, 0, -1, DBL_MAX};
    if (accum[ns] - acc_new < h->p.distance_new_keyframe_thresh) { h->reports.push_back(rep); continue; }
    acc_new = accum[ns];
    const int nc = loop_find(h->p, h->last_edge, poses16, accum, keyframes, n_kf, ns, cand);
    rep.n_candidates = nc;
    if (nc == 0) { rep.decision = LSD_LOOP_NO_CANDIDATES; h->reports.push_back(rep); continue; }
    guesses.resize(16 * (size_t)nc);
    for (int i = 0; i < nc; i++) loop_guess(poses16 + 16 * (size_t)ns, poses16 + 16 * (size_t)cand[i], guesses.data() + 16 * (size_t)i);
    long long ln = 0; int rd = 0;
    lsd_status_t s = loop_coarse(h, ns, cand.data(), guesses.data(), nc, &ln, &rd);
    if (s) return s;
    // best candidate (:175-191): converged only; a later candidate with an equal score wins
    int best = -1;
    double best_score = DBL_MAX;
    for (int i = 0; i < nc; i++) {
      if (!h->lm[i].converged) continue;
      if (h->fitness[i] > best_score) continue;
      best_score = h->fitness[i];
      best = i;
    }
    rep.best_slot = best >= 0 ? cand[best] : -1;
    rep.best_score = best_score;
    if (best_score > 2.0 * h->p.fitness_score_thresh) { rep.decision = LSD_LOOP_COARSE_REJECT; h->reports.push_back(rep); continue; }
    // refinement (:198-219): guess = the NDT result as Eigen::Matrix4f
    lsd_reg* g = h->gicp;
    s = lsd_reg_set_target_dev(g, reinterpret_cast<const float*>(h->d_pool + h->kf_off[ns]), h->kf_n[ns]);
    if (!s) s = lsd_reg_set_source_dev(g, reinterpret_cast<const float*>(h->d_pool + h->kf_off[cand[best]]), h->kf_n[cand[best]]);
    if (s) return s;
    double gs[16];
    for (int i = 0; i < 16; i++) gs[i] = (double)(float)h->lm[best].x0[i];
    s = reg_align(g, gs);
    if (s < 0) return s;
    if (!g->converged) { rep.decision = LSD_LOOP_GICP_DIVERGED; h->reports.push_back(rep); continue; }
    double score = 0;
    s = lsd_reg_fitness(g, nullptr, h->p.fitness_score_max_range, &score);
    if (s) return s;
    if (score > h->p.fitness_score_thresh) { rep.decision = LSD_LOOP_GICP_REJECT; h->reports.push_back(rep); continue; }
    rep.decision = LSD_LOOP_FOUND;
    h->reports.push_back(rep);
    h->last_edge = accum[ns];
    lsd_loop_result_t res;
    memset(&res, 0, sizeof(res));
    res.key1 = ns; res.key2 = cand[best];
    for (int i = 0; i < 16; i++) res.relpose16[i] = (float)g->final_T[i];
    res.coarse_score = best_score; res.score = score; res.n_candidates = nc;
    // calc_information_matrix(key1->cloud, key2->cloud, relpose): calc_fitness_score with max_range = DBL_MAX
    double fit = 0;
    s = lsd_loop_fitness(h, ns, cand[best], res.relpose16, DBL_MAX, &fit, nullptr);
    if (s) return s;
    loop_information(fit, res.information36);
    if (*n_loops < cap) out[*n_loops] = res;
    (*n_loops)++;
  }
  return LSD_OK;
}

}  // extern "C"
