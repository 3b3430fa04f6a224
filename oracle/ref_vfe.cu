// TEST INFRASTRUCTURE ONLY — never linked into the product (liblsdreg.so).
//
// C-ABI wrapper around the UNMODIFIED reference detection voxelizer, compiled where it lies under
// /root/reference/sensor_driver/inference/voxelize by oracle/Makefile (nvcc, sm_90a) into oracle/_ref/libref_vfe.so:
//   * Preprocess::forward     preprocess_kernel.cu:56-101   (sliding window, motion compensation)
//   * Voxelization::forward   voxelization_kernel.cu:225-255 (hash voxelisation, mean, fp16)
// Runs only where a GPU is present (the `-m gpu` tests); pins lsd_vfe_* against the reference's own kernels.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstring>
#include <vector>

#include "preprocess.hpp"
#include "voxelization.hpp"

struct RefVfe {
  std::shared_ptr<Preprocess> pre;
  std::shared_ptr<Voxelization> vox;
  VoxelizationParameter vp;
  PreprocessParameter pp;
  cudaStream_t stream = nullptr;
};

extern "C" {

void* refvfe_create(const float* min_range3, const float* max_range3, const float* voxel_size3, int max_points_per_voxel, int max_voxels,
                    int max_points, int num_feature, int max_frame_num) {
  RefVfe* h = new RefVfe;
  h->vp.min_range = nvtype::Float3(min_range3[0], min_range3[1], min_range3[2]);
  h->vp.max_range = nvtype::Float3(max_range3[0], max_range3[1], max_range3[2]);
  h->vp.voxel_size = nvtype::Float3(voxel_size3[0], voxel_size3[1], voxel_size3[2]);
  h->vp.grid_size = VoxelizationParameter::compute_grid_size(h->vp.max_range, h->vp.min_range, h->vp.voxel_size);
  h->vp.num_feature = num_feature;
  h->vp.max_voxels = max_voxels;
  h->vp.max_points_per_voxel = max_points_per_voxel;
  h->vp.max_points = max_points;
  h->pp.max_points = max_points;
  h->pp.num_feature = num_feature;
  h->pp.max_frame_num = max_frame_num;
  cudaStreamCreate(&h->stream);
  h->pre = create_preprocess(h->pp);
  h->vox = create_voxelization(h->vp);
  return h;
}
void refvfe_destroy(void* p) {
  RefVfe* h = static_cast<RefVfe*>(p);
  h->pre.reset(); h->vox.reset();
  cudaStreamDestroy(h->stream);
  delete h;
}
int refvfe_accumulate(void* p, const float* points_host, int num_points, const float* motion16_host, int realtime) {
  RefVfe* h = static_cast<RefVfe*>(p);
  h->pre->forward(points_host, num_points, motion16_host, realtime != 0, h->stream);
  return h->pre->get_points_num();
}
int refvfe_get_points(void* p, float* out_host, int cap_points) {
  RefVfe* h = static_cast<RefVfe*>(p);
  const int n = h->pre->get_points_num();
  const int c = n < cap_points ? n : cap_points;
  if (c > 0) cudaMemcpy(out_host, h->pre->get_points(), (size_t)c * h->pp.num_feature * sizeof(float), cudaMemcpyDeviceToHost);
  return n;
}
int refvfe_voxelize(void* p, int order_zyx) {
  RefVfe* h = static_cast<RefVfe*>(p);
  h->vox->forward(h->pre->get_points(), h->pre->get_points_num(), order_zyx ? CoordinateOrder::ZYX : CoordinateOrder::XYZ, h->stream);
  return h->vox->num_voxels();
}
// features: fp16 [V, num_feature] (raw 16-bit words), indices: u32 [V, 4]
int refvfe_get_output(void* p, unsigned short* features_host, unsigned* indices_host) {
  RefVfe* h = static_cast<RefVfe*>(p);
  half* f = nullptr; unsigned* idx = nullptr;
  const unsigned v = h->vox->get_output(&f, &idx);
  if (v > 0) {
    cudaMemcpy(features_host, f, (size_t)v * h->vp.num_feature * sizeof(unsigned short), cudaMemcpyDeviceToHost);
    cudaMemcpy(indices_host, idx, (size_t)v * 4 * sizeof(unsigned), cudaMemcpyDeviceToHost);
  }
  return (int)v;
}
void refvfe_grid(void* p, int* g3) { RefVfe* h = static_cast<RefVfe*>(p); g3[0] = h->vp.grid_size.x; g3[1] = h->vp.grid_size.y; g3[2] = h->vp.grid_size.z; }

}  // extern "C"
