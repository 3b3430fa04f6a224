// TEST INFRASTRUCTURE ONLY — never linked into the product (liblsdreg.so).
//
// C-ABI wrapper around the UNMODIFIED reference sources, compiled where they lie under
// /root/reference by oracle/Makefile into oracle/_ref/libref_lio.so:
//   * faster_lio::IVox      slam/mapping/fastlio/include/ivox3d/ivox3d.h:31-112   (live LIO map)
//   * KD_TREE (ikd-Tree)    slam/mapping/fastlio/include/ikd-Tree/ikd_Tree.{h,cpp} (named oracle)
//   * esti_plane<float>     slam/mapping/fastlio/include/common_lib.h:236-268
// Only this wrapper and the PCL point-type shims (oracle/ref_shim) are ours.  Map point ids are
// carried through the reference code in the normal_x / normal_y fields (16 bits each, exactly
// representable as float) so neighbour *indices* can be compared, not just coordinates.
#include <pcl/point_types.h>
typedef pcl::PointXYZINormal PointType;  // ivox3d_node.hpp:59 expects a global PointType

#include <common_lib.h>  // reference: esti_plane, calc_dist, PointVector
#include <ivox3d/ivox3d.h>
#include <ikd-Tree/ikd_Tree.h>

#include <omp.h>
#include <cstdint>
#include <cstring>

using IVoxType = faster_lio::IVox<3, faster_lio::IVoxNodeType::DEFAULT, PointType>;

static inline PointType mk(const float* p, int id) {
  PointType q;
  q.x = p[0]; q.y = p[1]; q.z = p[2];
  q.normal_x = float(id & 0xFFFF);
  q.normal_y = float((id >> 16) & 0xFFFF);
  return q;
}
static inline int id_of(const PointType& p) { return int(p.normal_x) | (int(p.normal_y) << 16); }

extern "C" {

// ---------------------------------------------------------------- iVox
void* ref_ivox_create(float res, int nearby, size_t capacity, double max_distance) {
  IVoxType::Options o;
  o.resolution_ = res;
  o.capacity_ = capacity;
  o.max_distance_ = max_distance;
  switch (nearby) {
    case 0: o.nearby_type_ = IVoxType::NearbyType::CENTER; break;
    case 6: o.nearby_type_ = IVoxType::NearbyType::NEARBY6; break;
    case 18: o.nearby_type_ = IVoxType::NearbyType::NEARBY18; break;
    case 26: o.nearby_type_ = IVoxType::NearbyType::NEARBY26; break;
    default: o.nearby_type_ = IVoxType::NearbyType::NEARBY74; break;
  }
  return new IVoxType(o);
}
void ref_ivox_destroy(void* h) { delete static_cast<IVoxType*>(h); }

void ref_ivox_add(void* h, const float* xyz, int n, int id0, double distance) {
  PointVector pv;
  pv.reserve(n);
  for (int i = 0; i < n; i++) pv.push_back(mk(xyz + 3 * i, id0 + i));
  static_cast<IVoxType*>(h)->AddPoints(pv, distance);
}
// AddPoints with explicit ids (the LIO front-end's two calls per scan carry ids that are not one run id0 + i)
void ref_ivox_add_ids(void* h, const float* xyz, const int* ids, int n, double distance) {
  PointVector pv;
  pv.reserve(n);
  for (int i = 0; i < n; i++) pv.push_back(mk(xyz + 3 * i, ids[i]));
  static_cast<IVoxType*>(h)->AddPoints(pv, distance);
}
size_t ref_ivox_num_cells(void* h) { return static_cast<IVoxType*>(h)->NumValidGrids(); }
size_t ref_ivox_num_points(void* h) {
  IVoxType::PointVector all;
  static_cast<IVoxType*>(h)->GetAllPoints(all);
  return all.size();
}
// Every stored point (IVox::GetAllPoints: voxel by voxel, each voxel's points in insertion order) with its voxel key.
// The key is Pos2Grid's own expression (ivox3d.h:259), evaluated here so that Eigen's rounding (half away from zero) and
// its float -> int conversion are the reference's; `res` is the resolution the map was created with, and the inverse is
// formed as the constructor forms options_.inv_resolution_ (ivox3d.h:58).  Returns the number of points; writes at most cap.
size_t ref_ivox_dump(void* h, float res, int* key3, float* xyz, int* ids, size_t cap) {
  IVoxType::PointVector all;
  static_cast<IVoxType*>(h)->GetAllPoints(all);
  const float inv = 1.0 / res;
  for (size_t i = 0; i < all.size() && i < cap; i++) {
    const Eigen::Matrix<float, 3, 1> p(all[i].x, all[i].y, all[i].z);
    const Eigen::Matrix<int, 3, 1> k = (p * inv).array().round().template cast<int>();
    for (int d = 0; d < 3; d++) { key3[3 * i + d] = k(d); xyz[3 * i + d] = (&all[i].x)[d]; }
    ids[i] = id_of(all[i]);
  }
  return all.size();
}
// IVox::SetNearByType (ivox3d.h:64-67): the pipeline starts on NEARBY74 and switches to NEARBY18 (laserMapping.cpp:1241-1243)
void ref_ivox_set_nearby(void* h, int nearby) {
  IVoxType::NearbyType t = IVoxType::NearbyType::NEARBY74;
  switch (nearby) {
    case 0: t = IVoxType::NearbyType::CENTER; break;
    case 6: t = IVoxType::NearbyType::NEARBY6; break;
    case 18: t = IVoxType::NearbyType::NEARBY18; break;
    case 26: t = IVoxType::NearbyType::NEARBY26; break;
    default: break;
  }
  static_cast<IVoxType*>(h)->SetNearByType(t);
}

// k-NN exactly as laserMapping.cpp:849 calls it.  out_ids [nq,k] (-1 padded), out_xyz [nq,k,3],
// out_cnt [nq].  Order within a row is the reference's (nearest first, rest nth_element order).
void ref_ivox_knn(void* h, const float* q, int nq, int k, double max_sq, int* out_ids, float* out_xyz,
                  int* out_cnt, int nthreads) {
  IVoxType* iv = static_cast<IVoxType*>(h);
  omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < nq; i++) {
    PointType p = mk(q + 3 * i, 0);
    PointVector near;
    iv->GetClosestPoint(p, near, k, max_sq);
    int c = int(near.size());
    out_cnt[i] = c;
    for (int j = 0; j < k; j++) {
      out_ids[i * k + j] = j < c ? id_of(near[j]) : -1;
      for (int d = 0; d < 3; d++) out_xyz[(i * k + j) * 3 + d] = j < c ? (&near[j].x)[d] : 0.f;
    }
  }
}

// ---------------------------------------------------------------- ikd-Tree
void* ref_ikd_create() { return new KD_TREE<PointType>(); }  // heap: 1M-entry op log inside
void ref_ikd_destroy(void* h) { delete static_cast<KD_TREE<PointType>*>(h); }
void ref_ikd_build(void* h, const float* xyz, int n, int id0) {
  PointVector pv;
  pv.reserve(n);
  for (int i = 0; i < n; i++) pv.push_back(mk(xyz + 3 * i, id0 + i));
  static_cast<KD_TREE<PointType>*>(h)->Build(pv);
}
// Delete_Point_Boxes (ikd_Tree.cpp:536-556): boxes [n,6] = (min xyz, max xyz); returns the tree's own count
int ref_ikd_delete_boxes(void* h, const float* boxes, int n) {
  std::vector<BoxPointType> bv(n);
  for (int i = 0; i < n; i++) for (int a = 0; a < 3; a++) { bv[i].vertex_min[a] = boxes[6 * i + a]; bv[i].vertex_max[a] = boxes[6 * i + 3 + a]; }
  return static_cast<KD_TREE<PointType>*>(h)->Delete_Point_Boxes(bv);
}
// Nearest_Search as laserMapping.cpp:846; out_d2 [nq,k] are the tree's own float distances.
void ref_ikd_knn(void* h, const float* q, int nq, int k, int* out_ids, float* out_d2, int* out_cnt,
                 int nthreads) {
  KD_TREE<PointType>* t = static_cast<KD_TREE<PointType>*>(h);
  omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < nq; i++) {
    PointType p = mk(q + 3 * i, 0);
    PointVector near;
    std::vector<float> d2(k);
    t->Nearest_Search(p, k, near, d2);
    int c = int(near.size());
    out_cnt[i] = c;
    for (int j = 0; j < k; j++) {
      out_ids[i * k + j] = j < c ? id_of(near[j]) : -1;
      out_d2[i * k + j] = j < c ? d2[j] : -1.f;
    }
  }
}

// ---------------------------------------------------------------- esti_plane
// pts5: [n,5,3]; pabcd: [n,4]; ok: [n]
void ref_esti_plane(const float* pts5, int n, float thr, float* pabcd, int* ok) {
  for (int i = 0; i < n; i++) {
    PointVector pv(5);
    for (int j = 0; j < 5; j++) {
      pv[j].x = pts5[(i * 5 + j) * 3 + 0];
      pv[j].y = pts5[(i * 5 + j) * 3 + 1];
      pv[j].z = pts5[(i * 5 + j) * 3 + 2];
    }
    Eigen::Matrix<float, 4, 1> r;
    ok[i] = esti_plane(r, pv, thr) ? 1 : 0;
    for (int d = 0; d < 4; d++) pabcd[i * 4 + d] = r(d);
  }
}


// The factorisation esti_plane runs (common_lib.h:251: A.colPivHouseholderQr().solve(b)), with its intermediates exposed, so that
// the plain-C restatement can be pinned step by step: packed QR (column-major 5x3), Householder coefficients, column permutation,
// number of non-zero pivots, and the solution.  Same Eigen, same flags, same matrix types as esti_plane.
void ref_esti_plane_qr(const float* pts5, int n, float* qr15, float* hc3, int* perm3, int* nzp, float* x3) {
  for (int i = 0; i < n; i++) {
    Eigen::Matrix<float, 5, 3> A;
    Eigen::Matrix<float, 5, 1> b;
    A.setZero(); b.setOnes(); b *= -1.0f;
    for (int j = 0; j < 5; j++) for (int d = 0; d < 3; d++) A(j, d) = pts5[(i * 5 + j) * 3 + d];
    Eigen::ColPivHouseholderQR<Eigen::Matrix<float, 5, 3>> qr = A.colPivHouseholderQr();
    Eigen::Matrix<float, 3, 1> x = qr.solve(b);
    for (int c = 0; c < 3; c++) for (int r = 0; r < 5; r++) qr15[i * 15 + c * 5 + r] = qr.matrixQR()(r, c);
    for (int c = 0; c < 3; c++) { hc3[i * 3 + c] = qr.hCoeffs()(c); perm3[i * 3 + c] = qr.colsPermutation().indices()(c); x3[i * 3 + c] = x(c); }
    nzp[i] = (int)qr.nonzeroPivots();
  }
}

// std::nth_element exactly as IVox::GetClosestPoint / KNNPointByCondition call it: on a std::vector of the reference's own
// DistPoint (ivox3d_node.hpp:72-85, operator< on the distance alone), this toolchain's libstdc++.  idx_inout carries the
// payload (DistPoint::idx) so that the resulting permutation can be read back.
void ref_std_nth_element(const double* dist, int* idx_inout, int n, int first, int nth, int last) {
  typedef faster_lio::IVoxNode<PointType, 3>::DistPoint DP;
  std::vector<DP> v(n);
  for (int i = 0; i < n; i++) v[i] = DP(dist[idx_inout[i]], nullptr, idx_inout[i]);
  std::nth_element(v.begin() + first, v.begin() + nth, v.begin() + last);
  for (int i = 0; i < n; i++) idx_inout[i] = v[i].idx;
}

// ---------------------------------------------------------------- full h-model on reference classes
// Restates the loop of h_share_model_geometric (laserMapping.cpp:813-982) around the UNMODIFIED
// reference IVox::GetClosestPoint and esti_plane<float> (Eigen ColPivHouseholderQR), with Eigen's
// SelfAdjointEigenSolver for the degeneracy test exactly as the reference does.  Same signature as
// orc_lio_hmodel (oracle/lsd_oracle.c) so oracle/lio.py can drive either.
int ref_lio_hmodel(void* hv, const float* body, int n, const double* R_, const double* t_, const double* RL_,
                   const double* tL_, int search, int knn_mode, float* near_xyz, int* near_ids, int* near_cnt,
                   unsigned char* selected, float* world, float* plane, double* HTH, double* HTh, double* res_sum,
                   int* degenerate, int degenerate_detect_en, double* hx_out, double* h_out, int nthreads) {
  IVoxType* iv = static_cast<IVoxType*>(hv);
  Eigen::Map<const Eigen::Matrix<double, 3, 3, Eigen::RowMajor>> R(R_), RL(RL_);
  Eigen::Map<const V3D> t(t_), tL(tL_);
  omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < n; i++) {
    const float* pb = body + 4 * (size_t)i;
    V3D p_body(pb[0], pb[1], pb[2]);
    V3D p_global(R * (RL * p_body + tL) + t);
    PointType point_world;
    point_world.x = p_global(0); point_world.y = p_global(1); point_world.z = p_global(2);
    float* w = world + 4 * (size_t)i;
    w[0] = point_world.x; w[1] = point_world.y; w[2] = point_world.z; w[3] = pb[3];
    PointVector points_near;
    if (search) {
      iv->GetClosestPoint(point_world, points_near, NUM_MATCH_POINTS, 5);
      int c = int(points_near.size());
      // knn_mode & 2: keep row i's previous list when GetClosestPoint found no candidate (it returns before clear(),
      // ivox3d.h:155-157, and the reference's Nearest_Points[i] outlives the scan, laserMapping.cpp:1273)
      if (!((knn_mode & 2) && c == 0)) {
        near_cnt[i] = c;
        for (int j = 0; j < 5; j++) {
          near_ids[5 * (size_t)i + j] = j < c ? id_of(points_near[j]) : -1;
          for (int d = 0; d < 3; d++) near_xyz[(5 * (size_t)i + j) * 3 + d] = j < c ? (&points_near[j].x)[d] : 0.f;
        }
      }
      selected[i] = near_cnt[i] >= NUM_MATCH_POINTS;
      if (selected[i] && c == 0) {
        points_near.resize(5);
        for (int j = 0; j < 5; j++) for (int d = 0; d < 3; d++) (&points_near[j].x)[d] = near_xyz[(5 * (size_t)i + j) * 3 + d];
      }
    } else if (selected[i]) {
      points_near.resize(5);
      for (int j = 0; j < 5; j++) for (int d = 0; d < 3; d++) (&points_near[j].x)[d] = near_xyz[(5 * (size_t)i + j) * 3 + d];
    }
    if (!selected[i]) continue;
    VF(4) pabcd;
    selected[i] = 0;
    if (esti_plane(pabcd, points_near, 0.1f)) {
      float pd2 = pabcd(0) * point_world.x + pabcd(1) * point_world.y + pabcd(2) * point_world.z + pabcd(3);
      float s = 1 - 0.9 * fabs(pd2) / sqrt(p_body.norm());
      if (s > 0.9) {
        selected[i] = 1;
        float* pl = plane + 4 * (size_t)i;
        pl[0] = pabcd(0); pl[1] = pabcd(1); pl[2] = pabcd(2); pl[3] = pd2;
      }
    }
  }
  int ne = 0;
  double total = 0.0;
  for (int i = 0; i < n; i++) if (selected[i]) { total += std::abs(plane[4 * (size_t)i + 3]); ne++; }
  *res_sum = total; *degenerate = 0;
  memset(HTH, 0, sizeof(double) * 36); memset(HTh, 0, sizeof(double) * 6);
  if (ne < 1) return 0;
  Eigen::MatrixXd h_x = Eigen::MatrixXd::Zero(ne, 6);
  Eigen::VectorXd h(ne);
  int k = 0;
  for (int i = 0; i < n; i++) {
    if (!selected[i]) continue;
    const float* pb = body + 4 * (size_t)i; const float* pl = plane + 4 * (size_t)i;
    V3D point_this_be(pb[0], pb[1], pb[2]);
    V3D point_this = RL * point_this_be + tL;
    M3D point_crossmat;
    point_crossmat << SKEW_SYM_MATRX(point_this);
    V3D norm_vec(pl[0], pl[1], pl[2]);
    V3D C(R.transpose() * norm_vec);
    V3D A(point_crossmat * C);
    h_x.row(k) << pl[0], pl[1], pl[2], A(0), A(1), A(2);
    h(k) = -pl[3];
    k++;
  }
  if (degenerate_detect_en) {  // laserMapping.cpp:934-980
    Eigen::MatrixXd hn = h_x.leftCols(3);
    Eigen::Matrix<double, 3, 3> H3 = hn.transpose() * hn;
    Eigen::SelfAdjointEigenSolver<Eigen::Matrix<double, 3, 3>> esolver(H3);
    Eigen::Matrix<double, 3, 3> mat_v = esolver.eigenvectors().real();
    Eigen::Matrix<double, 3, 3> mat_v2 = mat_v.transpose();
    bool deg = false;
    for (int i = 0; i < 3; i++) {
      float local_contri = 0, local_strong = 0;
      for (int j = 0; j < ne; j++) {
        V3D feat_row = hn.row(j).transpose();
        feat_row.normalize();
        V3D dir = mat_v.col(i);
        const float dotp = fabs(feat_row.dot(dir));
        if (dotp > 0.1736) local_contri += dotp;
        if (dotp > 0.7070) local_strong += dotp;
      }
      if (local_contri < 250.0 && local_strong < 50.0) { for (int j = 0; j < 3; j++) mat_v2(i, j) = 0; deg = true; }
    }
    if (deg) {
      Eigen::Matrix<double, 3, 3> mat_p = mat_v.transpose().inverse() * mat_v2;
      h_x.leftCols(3) = (mat_p * hn.transpose()).transpose();
      *degenerate = 1;
    }
  }
  Eigen::Matrix<double, 6, 6> M = h_x.transpose() * h_x;
  Eigen::Matrix<double, 6, 1> v = h_x.transpose() * h;
  for (int a = 0; a < 6; a++) { for (int b = 0; b < 6; b++) HTH[6 * a + b] = M(a, b); HTh[a] = v(a); }
  if (hx_out) for (int r = 0; r < ne; r++) for (int c = 0; c < 6; c++) hx_out[6 * (size_t)r + c] = h_x(r, c);
  if (h_out) for (int r = 0; r < ne; r++) h_out[r] = h(r);
  return ne;
}

// map_incremental (laserMapping.cpp:523-576) feeding the reference IVox::AddPoints.
int ref_map_incremental(void* hv, const float* body, int n, const double* R_, const double* t_, const double* RL_,
                        const double* tL_, const float* near_xyz, const int* near_cnt, int ekf_inited, double fsize,
                        float* world, unsigned char* flag, int id0, int id_t2) {
  IVoxType* iv = static_cast<IVoxType*>(hv);
  Eigen::Map<const Eigen::Matrix<double, 3, 3, Eigen::RowMajor>> R(R_), RL(RL_);
  Eigen::Map<const V3D> t(t_), tL(tL_);
  PointVector PointToAdd, PointNoNeedDownsample;
  for (int i = 0; i < n; i++) {
    const float* pb = body + 4 * (size_t)i;
    V3D p_body(pb[0], pb[1], pb[2]);
    V3D p_global(R * (RL * p_body + tL) + t);
    PointType pw = mk(pb, id0 + i);
    pw.x = p_global(0); pw.y = p_global(1); pw.z = p_global(2);
    float* w = world + 4 * (size_t)i;
    w[0] = pw.x; w[1] = pw.y; w[2] = pw.z; w[3] = pb[3];
    int f = 1;
    if (near_cnt[i] > 0 && ekf_inited) {
      PointType mid_point, n0;
      const float* nr = near_xyz + 15 * (size_t)i;
      n0.x = nr[0]; n0.y = nr[1]; n0.z = nr[2];
      mid_point.x = floor(pw.x / fsize) * fsize + 0.5 * fsize;
      mid_point.y = floor(pw.y / fsize) * fsize + 0.5 * fsize;
      mid_point.z = floor(pw.z / fsize) * fsize + 0.5 * fsize;
      float dist = calc_dist(pw, mid_point);
      if (fabs(n0.x - mid_point.x) > 0.5 * fsize && fabs(n0.y - mid_point.y) > 0.5 * fsize && fabs(n0.z - mid_point.z) > 0.5 * fsize) {
        f = 2;
      } else {
        for (int r = 0; r < NUM_MATCH_POINTS; r++) {
          if (near_cnt[i] < NUM_MATCH_POINTS) break;
          PointType q; q.x = nr[3 * r]; q.y = nr[3 * r + 1]; q.z = nr[3 * r + 2];
          if (calc_dist(q, mid_point) < dist) { f = 0; break; }
        }
      }
    }
    flag[i] = (unsigned char)f;
    if (f == 2 && id_t2) { PointType p2 = mk(pb, id0 + i + id_t2); p2.x = pw.x; p2.y = pw.y; p2.z = pw.z; pw = p2; }   // label only: ids in insertion order
    if (f == 1) PointToAdd.push_back(pw); else if (f == 2) PointNoNeedDownsample.push_back(pw);
  }
  iv->AddPoints(PointToAdd, 0.0);
  iv->AddPoints(PointNoNeedDownsample, 0.0);
  return int(PointToAdd.size() + PointNoNeedDownsample.size());
}


// so3_math.h:36-58  Exp(ang_vel, dt) — the rotation used by the per-point undistortion (IMU_Processing.hpp:384).
// common_lib.h already pulled the reference header in; out9 is row-major.
void ref_so3_exp(const double* ang_vel3, double dt, double* out9) {
  const Eigen::Vector3d w(ang_vel3[0], ang_vel3[1], ang_vel3[2]);
  const Eigen::Matrix3d R = Exp(w, dt);
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) out9[3 * a + b] = R(a, b);
}

}  // extern "C"
