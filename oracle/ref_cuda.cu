// TEST INFRASTRUCTURE ONLY — never linked into the product (liblsdreg.so).
//
// C-ABI wrapper around the UNMODIFIED reference CUDA matcher, compiled where it lies under
// /root/reference/slam/thirdparty/fast_gicp by oracle/Makefile (nvcc, sm_90a) into oracle/_ref/libref_cuda.so:
//   * fast_gicp::cuda::NDTCudaCore + its kernels   src/fast_gicp/cuda/{ndt_cuda,gaussian_voxelmap,
//         find_voxel_correspondences,ndt_compute_derivatives,covariance_regularization}.cu
//   * fast_gicp::NDTCuda (LsqRegistration LM loop)  include/fast_gicp/ndt/impl/ndt_cuda_impl.hpp,
//                                                  include/fast_gicp/gicp/impl/lsq_registration_impl.hpp
// It needs a GPU to run, so it is used by the `-m gpu` tests and by bench_extra.py's "reference kernels" leg:
// the reference's own CUDA code, recompiled for sm_90a, on the same H100 as liblsdreg.
// PCL / Boost are shimmed exactly as for oracle/ref_reg.cpp (oracle/ref_shim_reg, ours).
#include <pcl/point_types.h>
#include <pcl/point_cloud.h>
#include <pcl/registration/registration.h>

#include <fast_gicp/ndt/ndt_cuda.hpp>
#include <fast_gicp/gicp/impl/lsq_registration_impl.hpp>
#include <fast_gicp/ndt/impl/ndt_cuda_impl.hpp>
#include <fast_gicp/cuda/gaussian_voxelmap.cuh>

#include <cstring>

using P = pcl::PointXYZI;
using Cloud = pcl::PointCloud<P>;

struct NdtX : fast_gicp::NDTCuda<P, P> {
  using fast_gicp::NDTCuda<P, P>::linearize;
  using fast_gicp::NDTCuda<P, P>::compute_error;
  fast_gicp::cuda::NDTCudaCore* core() { return ndt_cuda_.get(); }
};

struct RefNdt {
  std::shared_ptr<NdtX> r;
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

// registrations.cpp:107-118: P2D, DIRECT7, resolution 1.0, 64 iterations, eps 0.01 / 0.1 deg
void* refndt_create(double resolution, int neighbors, int max_iterations, double trans_eps, double rot_eps_deg) {
  RefNdt* h = new RefNdt;
  h->r.reset(new NdtX);
  h->r->setDistanceMode(fast_gicp::NDTDistanceMode::P2D);
  h->r->setResolution(resolution);
  h->r->setNeighborSearchMethod(neighbors == 27 ? fast_gicp::NeighborSearchMethod::DIRECT27
                                : neighbors == 1 ? fast_gicp::NeighborSearchMethod::DIRECT1 : fast_gicp::NeighborSearchMethod::DIRECT7);
  h->r->setMaximumIterations(max_iterations);
  h->r->setTransformationEpsilon(trans_eps);
  h->r->setRotationEpsilon(rot_eps_deg);
  return h;
}
void refndt_destroy(void* h) { delete static_cast<RefNdt*>(h); }
void refndt_set_source(void* h, const float* xyz, int n, int stride) {
  RefNdt* r = static_cast<RefNdt*>(h);
  r->src = mk_cloud(xyz, n, stride);
  r->r->setInputSource(r->src);
}
void refndt_set_target(void* h, const float* xyz, int n, int stride) {
  RefNdt* r = static_cast<RefNdt*>(h);
  r->tgt = mk_cloud(xyz, n, stride);
  r->r->setInputTarget(r->tgt);
}
int refndt_num_voxels(void* h) {
  auto* c = static_cast<RefNdt*>(h)->r->core();
  return c->target_voxelmap ? c->target_voxelmap->voxelmap_info.num_voxels : 0;
}
// linearize(T): update_correspondences + compute_error with derivatives (H36 / b6 may be NULL)
double refndt_linearize(void* h, const double* T16, double* H36, double* b6) {
  RefNdt* r = static_cast<RefNdt*>(h);
  Eigen::Matrix<double, 6, 6> H; Eigen::Matrix<double, 6, 1> b;
  const double e = H36 ? r->r->linearize(iso(T16), &H, &b) : r->r->linearize(iso(T16), nullptr, nullptr);
  if (H36) for (int a = 0; a < 6; a++) { for (int c = 0; c < 6; c++) H36[6 * a + c] = H(a, c); b6[a] = b(a); }
  return e;
}
double refndt_compute_error(void* h, const double* T16) { return static_cast<RefNdt*>(h)->r->compute_error(iso(T16)); }
int refndt_num_correspondences(void* h) {
  auto* c = static_cast<RefNdt*>(h)->r->core();
  return c->correspondences ? (int)c->correspondences->size() : 0;
}
int refndt_align(void* h, const float* guess16, float* out16) {
  RefNdt* r = static_cast<RefNdt*>(h);
  Eigen::Matrix4f g;
  for (int a = 0; a < 4; a++) for (int b = 0; b < 4; b++) g(a, b) = guess16[4 * a + b];
  Cloud out;
  r->r->align(out, g);
  const Eigen::Matrix4f T = r->r->getFinalTransformation();
  for (int a = 0; a < 4; a++) for (int b = 0; b < 4; b++) out16[4 * a + b] = T(a, b);
  return r->r->hasConverged() ? 1 : 0;
}

}  // extern "C"
