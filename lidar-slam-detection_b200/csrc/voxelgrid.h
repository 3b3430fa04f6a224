// voxelgrid.h — host-side handle of the voxel-grid downsampler (K1).
#pragma once
#include <algorithm>

#include "lsd_common.cuh"

namespace lsd {
struct VgGrid {  // device-resident grid description, written by vg_setup_kernel
  float inv;
  int minb[3], divb[3], mul[3];
  int n_words;
  int status;  // 0, LSD_ERR_GRID_OVERFLOW (PCL: output = input) or LSD_ERR_CAPACITY
};
}  // namespace lsd

struct lsd_voxelgrid {
  int device = 0, max_points = 0, scan_blocks = 0, coop_blocks = lsd::kNumSms;
  long long max_cells = 0;
  cudaStream_t stream = nullptr;
  int* bbox = nullptr;            // ordered-int min[3], max[3]
  lsd::VgGrid* grid = nullptr;
  unsigned* bitmap = nullptr;     // occupancy, 1 bit per leaf; all-zero between calls
  int* word_prefix = nullptr;     // exclusive popcount prefix inside a scan chunk
  int* chunk_sum = nullptr;       // chunk totals -> exclusive chunk offsets
  int* vidx = nullptr;            // leaf index per input point
  int* out_vidx = nullptr;        // leaf index per output point
  long long* sums = nullptr;      // [max_points,4] fixed-point channel sums; all-zero between calls
  int* cnt = nullptr;
  int *off = nullptr, *slot = nullptr, *seg = nullptr;   // input-order sums: leaf offsets [m+1], each point's place in its leaf's segment, members
  int *crowd = nullptr, *crowd_n = nullptr;               // crowded leaves (front) and big leaves (back) and their numbers (written by every call)
  int input_order_sums = 1;       // centroids as pcl::VoxelGrid's sequential fp32 sums in input order (LSD_VG_SUMS=fixed: exact fixed-point sums)
  float4 *io_in = nullptr, *io_out = nullptr;  // staging for the host-pointer entry point
  int* d_m = nullptr;
  unsigned* done = nullptr;       // last-block tickets: [0] vg_scan_kernel, [1] vg_count_kernel
  long long launches = 0;
  int pdl = 0;                    // launch the kernels with programmatic dependent launch (lsd_lio_set_pdl)
};

namespace lsd {
lsd_status_t vg_run(lsd_voxelgrid* g, const float4* d_in, int n, float leaf, float4* d_out, int* d_m, cudaStream_t st);
inline int vg_launches(const lsd_voxelgrid* g) { return g->input_order_sums ? 6 : 5; }   // kernels per vg_run with n > 0
}
