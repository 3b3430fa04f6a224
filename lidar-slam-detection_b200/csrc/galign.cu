// galign.cu — the closure search of global_alignment (slam/localization/include/global_alignment.hpp:200-258) with its
// FAST_VGICP stage batched over every (new key frame, reference key frame) pair.
//
// The reference aligns the ScanContext matches of each new key frame one after another (:229-254), each with
// LsqRegistration's Levenberg-Marquardt loop: one cost evaluation, one host round trip, and a setInputTarget that rebuilds
// the reference key frame's covariances and voxel map every time.  Here every reference key frame's tables are built once
// and kept, and every pair keeps its own LM state (LmState, reg.cu); the states advance together: one
// vgicp_cost_batch_kernel launch per round evaluates the next cost of every live pair, each against its own reference
// key frame's voxel table.  Per pair the launch is the single-pair launch of vgicp_cost_kernel: reg_grid(n) blocks with
// the same point-to-block partition, the same per-point body (vgicp_point, reg.cu), the same block_partials<29> and a
// last-block fold in grid_finalize's order (loop_finalize, loop.cu) — H, b, err and the correspondence count are the bits
// of vgicp_cost_kernel on the same tables.  The fitness launch runs lsd_reg_fitness's body (fitness_range) per pair
// against the pair's reference point map.  Included by lsdreg.cu after reg.cu, loop.cu and scancontext.cu.
#include <cmath>
#include <map>

namespace lsd {

// One pair of a batched launch: the reference key frame's tables, where the new key frame's points and the pair's
// correspondences are, and what to evaluate.
struct GaCand {
  VgView vg;             // cost: the reference key frame's VGICP voxel table
  MapView mv;            // fitness: the reference key frame's point map
  Pose34d T;             // cost: evaluation pose (linearisation pose when update)
  Pose34f Tf;            // fitness: the pose, in float as getFitnessScore applies it
  long long corr_off;    // cost: [n_off, n] correspondence slots and 6 [n_off, n] Mahalanobis doubles at this offset of the pools
  int src_off, n;        // new key frame: first point in the pool (and first covariance), point count
  int blk_off, n_blk;    // first block of the launch, blocks it gets (the single-pair grid for n)
  int row;               // result row (pair index in the caller's list)
  int update, deriv;     // cost: linearize (refresh correspondences and Mahalanobis matrices) / accumulate H and b
  int warp_shape;        // fitness: fitness_range<true> (one warp per point) instead of <false>, as lsd_reg_fitness
};

// One VGICP cost evaluation for every pair of the launch, each against its own reference key frame.
__global__ void __launch_bounds__(256) vgicp_cost_batch_kernel(const float4* __restrict__ pool, const double* __restrict__ nrm_pool,
                                                               const GaCand* __restrict__ cands, int n_cand, int n_off,
                                                               int* __restrict__ corr_pool, double* __restrict__ maha_pool,
                                                               double* __restrict__ partials, unsigned* __restrict__ done,
                                                               double* __restrict__ result, double seq) {
  const int c = loop_cand_of_block(cands, n_cand);
  const int n = cands[c].n, G = cands[c].n_blk, lb = (int)blockIdx.x - cands[c].blk_off;
  const bool update = cands[c].update != 0, deriv = cands[c].deriv != 0;
  const VgView v = cands[c].vg;
  const Pose34d T = cands[c].T;
  const float4* src = pool + cands[c].src_off;
  const double* src_nrm = nrm_pool + 4 * (size_t)cands[c].src_off;
  int* corr = corr_pool + cands[c].corr_off;
  double* maha = maha_pool + 6 * cands[c].corr_off;
  double vals[29];
#pragma unroll
  for (int j = 0; j < 29; j++) vals[j] = 0.0;
#pragma unroll 1
  for (int i = lb * blockDim.x + threadIdx.x; i < n; i += G * blockDim.x)
    vgicp_point(v, __ldg(src + i), src_nrm, i, n, n_off, T, corr, maha, update, deriv, vals);
  block_partials<29>(vals, partials);  // row blockIdx.x = blk_off + lb
  loop_finalize<29>(partials + (size_t)cands[c].blk_off * kNV, G, done + 1 + c, done, n_cand,
                    result + (size_t)(1 + cands[c].row) * kNV, result, seq);
}

// getFitnessScore(max_range) of every pair at its pose against its reference key frame's point map: per pair the shape,
// grid and body of lsd_reg_fitness (fitness_range, reg.cu) and its fold, so the same sum and count.
__global__ void __launch_bounds__(kRegWarps * 32, 2) fitness_pairs_kernel(const float4* __restrict__ pool, const GaCand* __restrict__ cands,
                                                                          int n_cand, float search_sq, float max_range,
                                                                          double* __restrict__ partials, unsigned* __restrict__ done,
                                                                          double* __restrict__ result, double seq) {
  const int c = loop_cand_of_block(cands, n_cand);
  const int n = cands[c].n, G = cands[c].n_blk, lb = (int)blockIdx.x - cands[c].blk_off;
  const MapView mv = cands[c].mv;
  const Pose34f Tf = cands[c].Tf;
  const float4* src = pool + cands[c].src_off;
  if (cands[c].warp_shape)  // block-uniform
    fitness_range<true>(mv, src, n, lb, G, Tf, search_sq, max_range, nullptr, 0, partials);
  else
    fitness_range<false>(mv, src, n, lb, G, Tf, search_sq, max_range, nullptr, 0, partials);
  loop_finalize<2>(partials + (size_t)cands[c].blk_off * kNV, G, done + 1 + c, done, n_cand,
                   result + (size_t)(1 + cands[c].row) * kNV, result, seq);
}

}  // namespace lsd

// ==================================================================== host side
struct lsd_galign {
  lsd_galign_params_t p{};
  int device = 0;
  // VGICP handle: owns the stream, the launch scratch of the single-pair kernels and the scratch point map of the new key
  // frames' covariances.  The serial path points its source / target fields at this handle's tables (GaBind).
  lsd_reg* r = nullptr;
  lsd_sc* sc = nullptr;      // ScanContext database of the reference key frames: index = reference index
  // key-frame pool: every cloud once, [sum n, 4] float, and its k-NN covariances [sum n, 4] double (built on first use)
  float4* d_pool = nullptr; double* d_nrm = nullptr; size_t pool_n = 0, pool_cap = 0;
  std::vector<size_t> kf_off;
  std::vector<int> kf_n, kf_ref;   // kf_ref: reference index, -1 for a new key frame
  std::vector<char> nrm_built;
  std::vector<int> ref_slot;       // reference index -> slot
  struct Target { lsd_map* map = nullptr; lsd::VgView vg{}; unsigned long long vg_lines = 0; bool built = false; };
  std::vector<Target> tgt;         // per slot; built for reference key frames on their first use as a target
  // batch scratch, grown to the largest batch seen
  lsd::BatchScratch<lsd::GaCand> b;
  int* d_corr = nullptr; double* d_maha = nullptr; size_t corr_cap = 0, maha_cap = 0;   // [n_off, n] slots / 6 doubles per pair
  int cost_new = -1, cost_ref = -1;                      // pair whose correspondences the scratch holds (lsd_galign_cost)
  // last lsd_galign_match / batch of lsd_galign_search
  std::vector<lsd::LmState> lm;
  std::vector<double> fitness;
  std::vector<lsd_galign_match_t> matches;               // last lsd_galign_search
  long long search_launches = 0; int search_rounds = 0, search_batches = 0;
};

namespace lsd {

struct GaPair { int new_slot, ref_slot; double guess[16]; };

static lsd_status_t ga_reserve(lsd_galign* h, const std::vector<GaPair>& pairs) {
  const int n_off = h->p.reg.ndt_neighbors;
  size_t rows = 0, corr = 0;
  for (const GaPair& q : pairs) {
    const int v = h->kf_n[q.new_slot];
    rows += (size_t)std::max(reg_grid(v), warp_grid(v));
    corr += (size_t)n_off * v;
  }
  lsd_status_t s = h->b.reserve((int)pairs.size(), rows);
  bool grown = false;
  if (!s) s = grow_dev(h->d_corr, h->corr_cap, corr, &grown);
  if (!s) s = grow_dev(h->d_maha, h->maha_cap, 6 * corr);
  if (grown) h->cost_new = h->cost_ref = -1;   // the correspondences lsd_galign_cost left are gone
  return s;
}

// The k-NN covariances of key frame `slot` (fast_gicp_impl.hpp:109-114), once; through the point map *mp.
static lsd_status_t ga_covariances(lsd_galign* h, int slot, lsd_map** mp) {
  if (h->nrm_built[slot]) return LSD_OK;
  lsd_reg* r = h->r;
  lsd_status_t s = gicp_covariances(r, mp, h->d_pool + h->kf_off[slot], h->kf_n[slot], h->d_nrm + 4 * h->kf_off[slot]);
  if (s) return s;
  LSD_CUDA(cudaStreamSynchronize(r->stream));
  h->nrm_built[slot] = 1;
  return LSD_OK;
}

// setInputTarget(keyframes[match.first]->mPoints) (:240) once per reference key frame: its point map (kept: fitness), its
// covariances and its voxel table — the steps of lsd_reg_set_target_dev (gicp_covariances, vgicp_voxel_table).
static lsd_status_t ga_target(lsd_galign* h, int slot) {
  lsd_galign::Target& t = h->tgt[slot];
  if (t.built) return LSD_OK;
  lsd_status_t s = ga_covariances(h, slot, &t.map);
  if (s) return s;
  s = vgicp_voxel_table(h->r, h->d_pool + h->kf_off[slot], h->d_nrm + 4 * h->kf_off[slot], h->kf_n[slot], t.vg, t.vg_lines);
  if (s) return s;
  t.built = true;
  return LSD_OK;
}

// Tables of every pair: reference key frames' targets, new key frames' covariances (through the handle's scratch map).
static lsd_status_t ga_prepare(lsd_galign* h, const std::vector<GaPair>& pairs) {
  for (const GaPair& q : pairs) {
    lsd_status_t s = ga_target(h, q.ref_slot);
    if (!s) s = ga_covariances(h, q.new_slot, &h->r->src_map);
    if (s) return s;
  }
  return LSD_OK;
}

// One batched launch of `na` cost candidates (b.h_cand) over `blocks` blocks; row 1 + i of b.h_res = pair i.
static lsd_status_t ga_cost_launch(lsd_galign* h, int na, int blocks) {
  cudaStream_t st = h->r->stream;
  double seq = 0;
  lsd_status_t s = h->b.upload(na, st, &seq);
  if (s) return s;
  vgicp_cost_batch_kernel<<<blocks, 256, 0, st>>>(h->d_pool, h->d_nrm, h->b.d_cand, na, h->p.reg.ndt_neighbors, h->d_corr, h->d_maha,
                                                  h->b.d_partials, h->b.d_done, h->b.d_res, seq);
  LSD_CUDA(cudaGetLastError());
  return h->b.wait(st, seq);
}

static void ga_cost_cand(const lsd_galign* h, GaCand& c, const GaPair& q, int row, int blk_off, long long corr_off, const double* T,
                         bool update, bool deriv) {
  memset(&c, 0, sizeof(c));
  c.vg = h->tgt[q.ref_slot].vg;
  c.src_off = (int)h->kf_off[q.new_slot]; c.n = h->kf_n[q.new_slot]; c.row = row;
  c.n_blk = reg_grid(c.n); c.blk_off = blk_off;
  c.corr_off = corr_off;
  c.update = update; c.deriv = deriv;
  T_to_pose(T, &c.T, nullptr);
}

// getFitnessScore(max_range) of every pair at poses[i], one launch; score[i] as getFitnessScore returns it.
static lsd_status_t ga_fitness(lsd_galign* h, const std::vector<GaPair>& pairs, const std::vector<const double*>& poses, double* score,
                               long long* launches) {
  const int n = (int)pairs.size();
  if (n == 0) return LSD_OK;
  int blocks = 0;
  for (int i = 0; i < n; i++) {
    GaCand& c = h->b.h_cand[i];
    memset(&c, 0, sizeof(c));
    c.mv = h->tgt[pairs[i].ref_slot].map->view;
    c.src_off = (int)h->kf_off[pairs[i].new_slot]; c.n = h->kf_n[pairs[i].new_slot]; c.row = i;
    c.warp_shape = c.n < kThreadShapeMin;
    c.n_blk = c.warp_shape ? warp_grid(c.n) : reg_grid(c.n);
    c.blk_off = blocks; blocks += c.n_blk;
    T_to_pose(poses[i], nullptr, &c.Tf);
  }
  cudaStream_t st = h->r->stream;
  double seq = 0;
  lsd_status_t s = h->b.upload(n, st, &seq);
  if (s) return s;
  const double max_range = h->p.fitness_score_max_range;
  fitness_pairs_kernel<<<blocks, kRegWarps * 32, 0, st>>>(h->d_pool, h->b.d_cand, n, fitness_search_sq(max_range, h->p.reg.map_resolution),
                                                          (float)max_range, h->b.d_partials, h->b.d_done, h->b.d_res, seq);
  LSD_CUDA(cudaGetLastError());
  (*launches)++;
  s = h->b.wait(st, seq);
  if (s) return s;
  for (int i = 0; i < n; i++) {
    const double sum = h->b.row(i)[0], cnt = h->b.row(i)[1];
    score[i] = cnt > 0 ? sum / cnt : DBL_MAX;
  }
  return LSD_OK;
}

// Every pair's LM loop of lsd_reg_align (registration->align(*aligned, init_guess), :242), advanced together, then
// getFitnessScore(fitness_score_max_range) of all of them in one launch.  Results in h->lm, h->fitness.
static lsd_status_t ga_batch(lsd_galign* h, const std::vector<GaPair>& pairs, long long* launches, int* rounds) {
  *launches = 0; *rounds = 0;
  const int n = (int)pairs.size();
  h->lm.assign(n, LmState());
  h->fitness.assign(n, 0.0);
  if (n == 0) return LSD_OK;
  const long long l0 = h->r->launches;
  lsd_status_t s = ga_prepare(h, pairs);
  if (!s) s = ga_reserve(h, pairs);
  if (s) return s;
  *launches += h->r->launches - l0;
  h->cost_new = h->cost_ref = -1;
  const int n_off = h->p.reg.ndt_neighbors;
  std::vector<long long> corr_off(n);
  long long co = 0;
  for (int i = 0; i < n; i++) { corr_off[i] = co; co += (long long)n_off * h->kf_n[pairs[i].new_slot]; }
  for (int i = 0; i < n; i++) lm_begin(h->lm[i], h->p.reg, pairs[i].guess);
  for (;;) {
    int na = 0, blocks = 0;
    for (int i = 0; i < n; i++) {
      const LmState& m = h->lm[i];
      if (m.done) continue;
      GaCand& c = h->b.h_cand[na++];
      ga_cost_cand(h, c, pairs[i], i, blocks, corr_off[i], m.want_T, m.want_update, m.want_update);
      blocks += c.n_blk;
    }
    if (na == 0) break;
    s = ga_cost_launch(h, na, blocks);
    if (s) return s;
    (*launches)++; (*rounds)++;
    for (int i = 0; i < n; i++) {
      LmState& m = h->lm[i];
      if (m.done) continue;
      const double* res = h->b.row(i);
      double H[36], b[6];
      if (m.want_update) unpack_hb(res, H, b);
      lm_feed(m, H, b, res[27]);
    }
  }
  std::vector<const double*> poses(n);
  for (int i = 0; i < n; i++) poses[i] = h->lm[i].x0;
  return ga_fitness(h, pairs, poses, h->fitness.data(), launches);
}

// The handle's lsd_reg pointed at (new key frame, reference key frame) tables of this handle, for the single-pair kernels;
// detached again when it goes out of scope, so lsd_reg_destroy never frees what the pool owns.
struct GaBind {
  lsd_reg* r;
  GaBind(lsd_galign* h, int new_slot, int ref_slot) : r(h->r) {
    const lsd_galign::Target& t = h->tgt[ref_slot];
    r->d_src = h->d_pool + h->kf_off[new_slot]; r->d_src_nrm = h->d_nrm + 4 * h->kf_off[new_slot]; r->n_src = h->kf_n[new_slot];
    r->d_tgt = h->d_pool + h->kf_off[ref_slot]; r->n_tgt = h->kf_n[ref_slot];
    r->tgt_map = t.map; r->tgt_map_built = true; r->vg = t.vg;
    r->d_corr = h->d_corr; r->d_maha = h->d_maha;
  }
  ~GaBind() {
    r->d_src = nullptr; r->d_src_nrm = nullptr; r->n_src = 0; r->d_tgt = nullptr; r->n_tgt = 0;
    r->tgt_map = nullptr; r->tgt_map_built = false; r->vg = VgView{}; r->d_corr = nullptr; r->d_maha = nullptr;
  }
};

// The same pairs one after another through lsd_reg_align's and lsd_reg_fitness's single-pair kernels on this handle's tables.
static lsd_status_t ga_serial(lsd_galign* h, const std::vector<GaPair>& pairs, long long* launches, int* rounds) {
  *launches = 0; *rounds = 0;
  const int n = (int)pairs.size();
  h->lm.assign(n, LmState());
  h->fitness.assign(n, 0.0);
  lsd_reg* r = h->r;
  const long long l0 = r->launches;
  lsd_status_t s = ga_prepare(h, pairs);
  if (s) return s;
  for (const GaPair& q : pairs) {   // one pair's scratch at a time
    s = ga_reserve(h, std::vector<GaPair>{q});
    if (s) return s;
  }
  h->cost_new = h->cost_ref = -1;
  for (int i = 0; i < n; i++) {
    GaBind bind(h, pairs[i].new_slot, pairs[i].ref_slot);
    const long long c0 = r->launches;
    s = reg_align(r, pairs[i].guess);
    if (s < 0) return s;
    *rounds += (int)(r->launches - c0);   // one vgicp_cost_kernel launch per cost evaluation
    LmState& m = h->lm[i];
    memcpy(m.x0, r->final_T, sizeof(m.x0));
    m.converged = r->converged; m.iterations = r->iterations; m.iter_log = r->iter_log;
    s = lsd_reg_fitness(r, nullptr, h->p.fitness_score_max_range, &h->fitness[i]);
    if (s) return s;
  }
  *launches = r->launches - l0;
  return LSD_OK;
}

// Eigen::Matrix4f yaw2matrix(const float& y) (Scancontext.cpp:68-75), widened to double
static void yaw_guess(float yaw, double* G) {
  const float c = std::cos(yaw), s = std::sin(yaw);
  for (int i = 0; i < 16; i++) G[i] = (i % 5 == 0) ? 1.0 : 0.0;
  G[0] = c; G[1] = -s; G[4] = s; G[5] = c;
}

static bool ga_slots_ok(const lsd_galign* h, const int32_t* s, int n, int want_ref) {
  for (int i = 0; i < n; i++) {
    if (s[i] < 0 || s[i] >= (int32_t)h->kf_n.size()) return false;
    if (want_ref >= 0 && (h->kf_ref[s[i]] >= 0) != (want_ref != 0)) return false;
  }
  return true;
}

}  // namespace lsd

using namespace lsd;

extern "C" {

void lsd_galign_default_params(lsd_galign_params_t* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  lsd_reg_default_params(&p->reg, LSD_REG_VGICP);   // select_registration_method("FAST_VGICP") (global_alignment.hpp:201)
  p->sc_dist_thres = 0.30;                          // global_alignment.hpp:31-34
  p->icp_score_thres = 1.5;
  p->fitness_score_max_range = 25.0;
  p->max_batch_points = 1ll << 24;
  p->sc_db_capacity = 4096;
}

lsd_status_t lsd_galign_create(lsd_galign_t** out, const lsd_galign_params_t* p) {
  if (!out || !p) return LSD_ERR_INVALID;
  if (p->reg.kind != LSD_REG_VGICP) { set_error("lsd_galign_create: the matcher is FAST_VGICP (global_alignment.hpp:201)"); return LSD_ERR_INVALID; }
  if (p->reg.max_process_time_us != 0) { set_error("lsd_galign_create: the matcher has no timeout"); return LSD_ERR_INVALID; }
  if (p->max_batch_points < 1 || p->sc_db_capacity < 1) { set_error("lsd_galign_create: max_batch_points and sc_db_capacity must be positive"); return LSD_ERR_INVALID; }
  lsd_galign* h = new lsd_galign();
  h->p = *p;
  lsd_status_t s = lsd_reg_create(&h->r, &p->reg);
  if (!s) s = lsd_sc_create(&h->sc, p->sc_db_capacity);
  if (s) { lsd_galign_destroy(h); return s; }
  h->device = h->r->device;
  *out = h;
  return LSD_OK;
}

lsd_status_t lsd_galign_destroy(lsd_galign_t* h) {
  if (!h) return LSD_OK;
  if (h->r) { cudaSetDevice(h->r->device); cudaStreamSynchronize(h->r->stream); }
  for (lsd_galign::Target& t : h->tgt) { if (t.map) lsd_map_destroy(t.map); cudaFree(t.vg.lines); }
  cudaFree(h->d_pool); cudaFree(h->d_nrm); cudaFree(h->d_corr); cudaFree(h->d_maha);
  h->b.release();
  lsd_reg_destroy(h->r);
  lsd_sc_destroy(h->sc);
  delete h;
  return LSD_OK;
}

lsd_status_t lsd_galign_add_keyframe(lsd_galign_t* h, const float* xyzi_host, int n, int reference, int32_t* slot) {
  if (!h || !xyzi_host || n <= 0) return LSD_ERR_INVALID;
  LSD_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->r->stream;
  if (h->pool_n + (size_t)n > (size_t)INT32_MAX) { set_error("lsd_galign_add_keyframe: key-frame pool above 2^31 points"); return LSD_ERR_CAPACITY; }
  if (reference) {
    int db = 0;
    lsd_sc_db_size(h->sc, &db);
    if (db >= h->p.sc_db_capacity) { set_error("lsd_galign_add_keyframe: %d reference key frames fill the ScanContext database (sc_db_capacity)", db); return LSD_ERR_CAPACITY; }
  }
  if (h->pool_n + (size_t)n > h->pool_cap) {
    const size_t cap = std::max(h->pool_n + (size_t)n, 2 * h->pool_cap);
    float4* np_ = nullptr; double* nn_ = nullptr;
    LSD_CUDA(cudaMalloc((void**)&np_, cap * 16));
    cudaError_t e = cudaMalloc((void**)&nn_, cap * 32);
    if (e != cudaSuccess) { cudaFree(np_); return cuda_fail(e, "lsd_galign_add_keyframe", __FILE__, __LINE__); }
    if (h->pool_n) {
      LSD_CUDA(cudaMemcpyAsync(np_, h->d_pool, h->pool_n * 16, cudaMemcpyDeviceToDevice, st));
      LSD_CUDA(cudaMemcpyAsync(nn_, h->d_nrm, h->pool_n * 32, cudaMemcpyDeviceToDevice, st));
    }
    LSD_CUDA(cudaStreamSynchronize(st));
    cudaFree(h->d_pool); cudaFree(h->d_nrm);
    h->d_pool = np_; h->d_nrm = nn_; h->pool_cap = cap;
  }
  LSD_CUDA(cudaMemcpyAsync(h->d_pool + h->pool_n, xyzi_host, (size_t)n * 16, cudaMemcpyHostToDevice, st));
  LSD_CUDA(cudaStreamSynchronize(st));
  const int32_t s = (int32_t)h->kf_n.size();
  if (reference) {   // KeyFrame's ScanContext (keyframe.cpp:165-167) into the database, in slot order
    lsd_status_t e = lsd_sc_make_dev(h->sc, reinterpret_cast<const float*>(h->d_pool + h->pool_n), n, nullptr, 1, nullptr, nullptr, nullptr);
    if (!e) e = lsd_sc_db_add_made(h->sc, 0);
    if (e) return e;
    h->ref_slot.push_back(s);
  }
  h->kf_off.push_back(h->pool_n); h->kf_n.push_back(n); h->kf_ref.push_back(reference ? (int)h->ref_slot.size() - 1 : -1);
  h->nrm_built.push_back(0);
  h->tgt.emplace_back();
  h->pool_n += (size_t)n;
  if (slot) *slot = s;
  return LSD_OK;
}

lsd_status_t lsd_galign_merge_candidates(const int32_t* cand_idx, const double* cand_dist, const int32_t* cand_shift,
                                         const int32_t* n_cand, int n_off, double dist_thres, int32_t* idx_out,
                                         float* dist_out, float* yaw_out, int cap, int* n_out) {
  if (!cand_idx || !cand_dist || !cand_shift || !n_cand || n_off < 0 || !n_out || (cap > 0 && (!idx_out || !dist_out || !yaw_out)))
    return LSD_ERR_INVALID;
  std::map<int, std::pair<float, float>> m;   // sc_idx -> (sc_dist, sc_yaw), global_alignment.hpp:207
  for (int o = 0; o < n_off; o++) {
    for (int c = 0; c < std::min((int)n_cand[o], (int)sc::kCand); c++) {
      const size_t at = (size_t)o * sc::kCand + c;
      if (!(cand_dist[at] < dist_thres)) continue;                        // detectCandidateMatch (Scancontext.cpp:354)
      const float d = (float)cand_dist[at], y = sc::shift_to_yaw(cand_shift[at]);
      auto it = m.find(cand_idx[at]);
      if (it == m.end() || it->second.first > d) m[cand_idx[at]] = {d, y};   // :222-226
    }
  }
  int k = 0;
  for (const auto& e : m) {
    if (k < cap) { idx_out[k] = e.first; dist_out[k] = e.second.first; yaw_out[k] = e.second.second; }
    k++;
  }
  *n_out = k;
  return LSD_OK;
}

lsd_status_t lsd_galign_search(lsd_galign_t* h, const int32_t* new_slots, int n_new, lsd_galign_closure_t* out, int cap,
                               int* n_closures) {
  if (!h || n_new < 0 || (n_new > 0 && !new_slots) || !n_closures || (cap > 0 && !out) || !ga_slots_ok(h, new_slots, n_new, 0)) {
    set_error("lsd_galign_search: bad slots (new key frames only) / arguments");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  *n_closures = 0;
  h->matches.clear();
  h->search_launches = 0; h->search_rounds = 0; h->search_batches = 0;
  // :209-227 for every new key frame: nine descriptors in one pass, one query, the merge
  static const double kSearchTrans[18] = {0, 0, -4, 0, 4, 0, 0, -4, 0, 4, -4, -4, -4, 4, 4, -4, 4, 4};
  const int n_off9 = 9;
  std::vector<std::vector<GaPair>> per_new(n_new);
  std::vector<std::vector<std::pair<float, float>>> sc_of(n_new);   // (sc_dist, sc_yaw) per pair
  std::vector<int32_t> idx(n_off9 * sc::kCand), sh(n_off9 * sc::kCand), nc(n_off9), m_idx(n_off9 * sc::kCand);
  std::vector<double> dist(n_off9 * sc::kCand);
  std::vector<float> m_dist(n_off9 * sc::kCand), m_yaw(n_off9 * sc::kCand);
  for (int q = 0; q < n_new; q++) {
    const int32_t ns = new_slots[q];
    lsd_status_t s = lsd_sc_make_dev(h->sc, reinterpret_cast<const float*>(h->d_pool + h->kf_off[ns]), h->kf_n[ns], kSearchTrans, n_off9,
                                     nullptr, nullptr, nullptr);
    if (!s) s = lsd_sc_query(h->sc, nullptr, n_off9, idx.data(), dist.data(), sh.data(), nc.data());
    int nm = 0;
    if (!s) s = lsd_galign_merge_candidates(idx.data(), dist.data(), sh.data(), nc.data(), n_off9, h->p.sc_dist_thres, m_idx.data(),
                                            m_dist.data(), m_yaw.data(), (int)m_idx.size(), &nm);
    if (s) return s;
    for (int k = 0; k < nm; k++) {
      GaPair pr;
      pr.new_slot = ns; pr.ref_slot = h->ref_slot[m_idx[k]];
      yaw_guess(-m_yaw[k], pr.guess);   // yaw2matrix(-match.second.sc_yaw) (:243)
      per_new[q].push_back(pr);
      sc_of[q].push_back({m_dist[k], m_yaw[k]});
    }
  }
  // batches of whole new key frames within max_batch_points; every pair runs the same whatever batch it is in
  const long long n_off = h->p.reg.ndt_neighbors;
  int q0 = 0;
  while (q0 < n_new) {
    std::vector<GaPair> pairs;
    long long used = 0;
    int q1 = q0;
    for (; q1 < n_new; q1++) {
      const long long need = n_off * h->kf_n[new_slots[q1]] * (long long)per_new[q1].size();
      if (q1 > q0 && used + need > h->p.max_batch_points) break;
      used += need;
      pairs.insert(pairs.end(), per_new[q1].begin(), per_new[q1].end());
    }
    long long ln = 0; int rd = 0;
    lsd_status_t s = ga_batch(h, pairs, &ln, &rd);
    if (s) return s;
    h->search_launches += ln; h->search_rounds += rd; h->search_batches++;
    int k = 0;
    for (int q = q0; q < q1; q++) {
      for (size_t j = 0; j < per_new[q].size(); j++, k++) {
        const LmState& m = h->lm[k];
        lsd_galign_match_t mt;
        memset(&mt, 0, sizeof(mt));
        mt.new_slot = pairs[k].new_slot; mt.ref_slot = pairs[k].ref_slot;
        mt.sc_dist = sc_of[q][j].first; mt.sc_yaw = sc_of[q][j].second;
        mt.converged = m.converged; mt.iterations = m.iterations; mt.score = h->fitness[k];
        mt.accepted = m.converged && h->fitness[k] < h->p.icp_score_thres;   // :245-253
        h->matches.push_back(mt);
        if (!mt.accepted) continue;
        if (*n_closures < cap) {
          lsd_galign_closure_t& c = out[*n_closures];
          memset(&c, 0, sizeof(c));
          c.ref_slot = mt.ref_slot; c.new_slot = mt.new_slot;
          for (int e = 0; e < 16; e++) c.relpose16[e] = (float)m.x0[e];   // getFinalTransformation (:250)
          c.score = mt.score; c.sc_dist = mt.sc_dist; c.sc_yaw = mt.sc_yaw;
        }
        (*n_closures)++;
      }
    }
    q0 = q1;
  }
  return LSD_OK;
}

lsd_status_t lsd_galign_set_max_batch_points(lsd_galign_t* h, int64_t max_batch_points) {
  if (!h || max_batch_points < 1) { set_error("lsd_galign_set_max_batch_points: must be positive"); return LSD_ERR_INVALID; }
  h->p.max_batch_points = max_batch_points;
  return LSD_OK;
}

lsd_status_t lsd_galign_last_matches(lsd_galign_t* h, lsd_galign_match_t* out, int cap, int* n) {
  if (!h || !n) return LSD_ERR_INVALID;
  *n = (int)h->matches.size();
  if (out) memcpy(out, h->matches.data(), (size_t)std::min(*n, std::max(cap, 0)) * sizeof(lsd_galign_match_t));
  return LSD_OK;
}

lsd_status_t lsd_galign_last_stats(lsd_galign_t* h, long long* launches, int* rounds, int* batches) {
  if (!h) return LSD_ERR_INVALID;
  if (launches) *launches = h->search_launches;
  if (rounds) *rounds = h->search_rounds;
  if (batches) *batches = h->search_batches;
  return LSD_OK;
}

lsd_status_t lsd_galign_match(lsd_galign_t* h, int32_t new_slot, const int32_t* ref_slots, const double* guesses16, int n,
                              int serial, double* final16, int32_t* converged, int32_t* iterations, double* fitness,
                              long long* launches, int* rounds) {
  if (!h || n < 0 || (n > 0 && (!ref_slots || !guesses16)) || !ga_slots_ok(h, &new_slot, 1, 0) || !ga_slots_ok(h, ref_slots, n, 1)) {
    set_error("lsd_galign_match: bad slots (one new key frame, reference key frames) / arguments");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  std::vector<GaPair> pairs(n);
  for (int i = 0; i < n; i++) {
    pairs[i].new_slot = new_slot; pairs[i].ref_slot = ref_slots[i];
    memcpy(pairs[i].guess, guesses16 + 16 * (size_t)i, 16 * sizeof(double));
  }
  long long ln = 0; int rd = 0;
  lsd_status_t s = serial ? ga_serial(h, pairs, &ln, &rd) : ga_batch(h, pairs, &ln, &rd);
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

lsd_status_t lsd_galign_iteration_log(lsd_galign_t* h, int i, double* out4_per_iter, int cap_iters, int* n_iters) {
  if (!h || !n_iters || i < 0 || i >= (int)h->lm.size()) return LSD_ERR_INVALID;
  const std::vector<double>& lg = h->lm[i].iter_log;
  const int n = (int)(lg.size() / 4);
  *n_iters = n;
  if (out4_per_iter) memcpy(out4_per_iter, lg.data(), (size_t)std::min(n, std::max(cap_iters, 0)) * 4 * sizeof(double));
  return LSD_OK;
}

lsd_status_t lsd_galign_cost(lsd_galign_t* h, int32_t new_slot, int32_t ref_slot, const double* T16, int update, double* H36,
                             double* b6, double* err, int* n_corr) {
  if (!h || !T16 || (H36 && !b6) || !ga_slots_ok(h, &new_slot, 1, 0) || !ga_slots_ok(h, &ref_slot, 1, 1)) {
    set_error("lsd_galign_cost: bad slots (a new and a reference key frame) / arguments");
    return LSD_ERR_INVALID;
  }
  if (!update && (h->cost_new != new_slot || h->cost_ref != ref_slot)) {
    set_error("lsd_galign_cost: compute_error needs a previous update of the same pair");
    return LSD_ERR_INVALID;
  }
  LSD_CUDA(cudaSetDevice(h->device));
  GaPair q;
  q.new_slot = new_slot; q.ref_slot = ref_slot;
  const std::vector<GaPair> pairs{q};
  lsd_status_t s = ga_prepare(h, pairs);
  if (!s) s = ga_reserve(h, pairs);
  if (s) return s;
  ga_cost_cand(h, h->b.h_cand[0], q, 0, 0, 0, T16, update != 0, H36 != nullptr);
  s = ga_cost_launch(h, 1, h->b.h_cand[0].n_blk);
  if (s) return s;
  h->cost_new = new_slot; h->cost_ref = ref_slot;
  const double* res = h->b.row(0);
  if (H36) unpack_hb(res, H36, b6);
  if (err) *err = res[27];
  if (n_corr) *n_corr = (int)(res[28] + 0.5);
  return LSD_OK;
}

}  // extern "C"
