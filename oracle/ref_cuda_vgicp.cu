// TEST INFRASTRUCTURE ONLY — never linked into the product (liblsdreg.so).
//
// C-ABI wrapper around the UNMODIFIED reference CUDA VGICP matcher — the method the reference selects by default where it
// is built with USE_VGICP_CUDA (hdl_graph_slam/registrations.cpp:25-27,43-55; global_localization.cpp:18;
// scan_matching_odometry_nodelet.cpp:122) — compiled where it lies under /root/reference/slam/thirdparty/fast_gicp by
// oracle/Makefile (nvcc, sm_90a) into oracle/_ref/libref_cuda_vgicp.so:
//   * fast_gicp::cuda::FastVGICPCudaCore + kernels   src/fast_gicp/cuda/{fast_vgicp_cuda,brute_force_knn,compute_derivatives,
//         compute_mahalanobis,covariance_estimation,covariance_estimation_rbf,covariance_regularization,gaussian_voxelmap,
//         find_voxel_correspondences}.cu
//   * fast_gicp::FastVGICPCuda (LsqRegistration LM loop)   include/fast_gicp/gicp/impl/{fast_vgicp_cuda_impl,lsq_registration_impl}.hpp
// Needs a GPU to run: used by the `-m gpu` comparator test and bench_extra.py's "reference kernels" leg (config 4, VGICP).
// PCL / Boost are shimmed exactly as for oracle/ref_reg.cpp (oracle/ref_shim_reg, ours).
#include <pcl/point_types.h>
#include <pcl/point_cloud.h>
#include <pcl/search/kdtree.h>
#include <pcl/registration/registration.h>

#include <fast_gicp/gicp/fast_vgicp_cuda.hpp>
#include <fast_gicp/gicp/impl/lsq_registration_impl.hpp>
#include <fast_gicp/gicp/impl/fast_vgicp_cuda_impl.hpp>

#include <cstring>

using P = pcl::PointXYZI;
using Cloud = pcl::PointCloud<P>;

struct VgX : fast_gicp::FastVGICPCuda<P, P> {
  using fast_gicp::FastVGICPCuda<P, P>::linearize;
  using fast_gicp::FastVGICPCuda<P, P>::compute_error;
};

struct RefVgicp {
  std::shared_ptr<VgX> r;
  Cloud::Ptr src, tgt;
};

static Cloud::Ptr mk_cloud(const float* xyz, int n, int stride) {
  Cloud::Ptr c(new Cloud);
  c->points.resize(n);
  for (int i = 0; i < n; i++) { P& p = c->points[i]; p.x = xyz[(size_t)stride * i]; p.y = xyz[(size_t)stride * i + 1]; p.z = xyz[(size_t)stride * i + 2]; p.w = 1.f; }
  return c;
}
static Eigen::Isometry3d iso(const double* T16) {
  Eigen::Isometry3d t = Eigen::Isometry3d::Identity();
  for (int a = 0; a < 3; a++) { for (int b = 0; b < 3; b++) t.linear()(a, b) = T16[4 * a + b]; t.translation()(a) = T16[4 * a + 3]; }
  return t;
}

extern "C" {

// registrations.cpp:43-55: resolution 1.0, eps 0.01, 64 iterations, k = 20; nn_method 0 = CPU_PARALLEL_KDTREE (the
// reference's setting), 1 = GPU_BRUTEFORCE, 2 = GPU_RBF_KERNEL
void* refvgicp_create(double resolution, int max_iterations, double trans_eps, int nn_method) {
  RefVgicp* h = new RefVgicp;
  h->r.reset(new VgX);
  h->r->setResolution(resolution);
  h->r->setTransformationEpsilon(trans_eps);
  h->r->setMaximumIterations(max_iterations);
  h->r->setCorrespondenceRandomness(20);
  h->r->setNearestNeighborSearchMethod(nn_method == 1 ? fast_gicp::NearestNeighborMethod::GPU_BRUTEFORCE
                                       : nn_method == 2 ? fast_gicp::NearestNeighborMethod::GPU_RBF_KERNEL
                                                        : fast_gicp::NearestNeighborMethod::CPU_PARALLEL_KDTREE);
  return h;
}
void refvgicp_destroy(void* h) { delete static_cast<RefVgicp*>(h); }
void refvgicp_set_source(void* h, const float* xyz, int n, int stride) {
  RefVgicp* r = static_cast<RefVgicp*>(h);
  r->src = mk_cloud(xyz, n, stride);
  r->r->setInputSource(r->src);
}
void refvgicp_set_target(void* h, const float* xyz, int n, int stride) {
  RefVgicp* r = static_cast<RefVgicp*>(h);
  r->tgt = mk_cloud(xyz, n, stride);
  r->r->setInputTarget(r->tgt);
}
// linearize(T): correspondences + error with derivatives (H36 / b6 may be NULL)
double refvgicp_linearize(void* h, const double* T16, double* H36, double* b6) {
  RefVgicp* r = static_cast<RefVgicp*>(h);
  Eigen::Matrix<double, 6, 6> H; Eigen::Matrix<double, 6, 1> b;
  const double e = H36 ? r->r->linearize(iso(T16), &H, &b) : r->r->linearize(iso(T16), nullptr, nullptr);
  if (H36) for (int a = 0; a < 6; a++) { for (int c = 0; c < 6; c++) H36[6 * a + c] = H(a, c); b6[a] = b(a); }
  return e;
}
double refvgicp_compute_error(void* h, const double* T16) { return static_cast<RefVgicp*>(h)->r->compute_error(iso(T16)); }
int refvgicp_align(void* h, const float* guess16, float* out16) {
  RefVgicp* r = static_cast<RefVgicp*>(h);
  Eigen::Matrix4f g;
  for (int a = 0; a < 4; a++) for (int b = 0; b < 4; b++) g(a, b) = guess16[4 * a + b];
  Cloud out;
  r->r->align(out, g);
  const Eigen::Matrix4f T = r->r->getFinalTransformation();
  for (int a = 0; a < 4; a++) for (int b = 0; b < 4; b++) out16[4 * a + b] = T(a, b);
  return r->r->hasConverged() ? 1 : 0;
}

}  // extern "C"
