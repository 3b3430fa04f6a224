/* lsdreg.h — C ABI of liblsdreg.so: the H100-native registration hot path for LSD.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point is `extern "C"`, takes plain
 * pointers and sizes, returns an `lsd_status_t` (0 = ok, < 0 = error, > 0 = informational), never
 * throws across the boundary, and cites the reference interface it replaces (paths relative to
 * /root/reference).  INTEGRATION.md shows the reference-side bindings (the C++ seams in
 * slam/mapping/fastlio/src/fastlio.cpp:9-16 and hdl_graph_slam/registrations.hpp:15-16, and the
 * pybind11 `slam_wrapper` module).
 *
 * Conventions
 *   - points are float32 [n,4] = (x, y, z, intensity), row-major, the layout py_utils.cpp:149-169
 *     hands to the reference;
 *   - `*_dev` variants take DEVICE pointers (inputs already resident in HBM) and never synchronise
 *     unless they must return a scalar; the plain variants take HOST pointers and include the
 *     H2D/D2H copies;
 *   - handles are confined to one thread at a time (SURVEY.md §8b "Thread-safety");
 *   - there is NO CPU fallback: every call fails with LSD_ERR_NO_DEVICE when no sm_90 GPU /
 *     CUDA driver is present.
 */
#ifndef LSDREG_H
#define LSDREG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int lsd_status_t;
#define LSD_OK 0
#define LSD_NO_EFFECTIVE_POINTS 1   /* ekfom_data.valid == false, laserMapping.cpp:888-893      */
#define LSD_SCAN_TOO_SMALL 2        /* feats_down_size < 5, laserMapping.cpp:1252-1256           */
#define LSD_MAP_SEEDED 3            /* first scan only seeded the map, laserMapping.cpp:1227-1239 */
#define LSD_LOCALMAP_NONE 5         /* Localization would set mLocalMap = nullptr (localization.cpp:352-364)                  */
#define LSD_MAP_SATURATED 6         /* the scan was registered, but the map refused points (lsd_map_saturated): enlarge map_log2_lines or enable the LRU */
#define LSD_IMU_INITIALIZING 4      /* ImuProcess::Process returned before undistorting (IMU_Processing.hpp:416-443) */
#define LSD_ERR_INVALID (-1)
#define LSD_ERR_CUDA (-2)
#define LSD_ERR_NO_DEVICE (-3)
#define LSD_ERR_CAPACITY (-4)       /* hash table / bucket levels / scratch capacity exceeded    */
#define LSD_ERR_GRID_OVERFLOW (-5)  /* voxel grid larger than int32 (PCL returns input unchanged) */
#define LSD_ERR_IO (-6)             /* key-frame file missing / unreadable / not the expected format */

const char* lsd_version(void);
const char* lsd_last_error(void);
/* Select the CUDA device for this thread's subsequent lsd_* calls (default 0). */
lsd_status_t lsd_init(int device);

/* ------------------------------------------------------------------------------------------
 * Hash-voxel map — replaces faster_lio::IVox (slam/mapping/fastlio/include/ivox3d/ivox3d.h:31-112:
 * AddPoints :231-256, GetClosestPoint :139-171, Pos2Grid :258-261) and, through the EXACT stencil,
 * the ikd-Tree queries (include/ikd-Tree/ikd_Tree.cpp:367-397 Nearest_Search).
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_map lsd_map_t;

/* stencils: IVox::NearbyType (ivox3d.h:40-46) + exact radius search */
#define LSD_STENCIL_CENTER 0
#define LSD_STENCIL_NEARBY6 6
#define LSD_STENCIL_NEARBY18 18
#define LSD_STENCIL_NEARBY26 26
#define LSD_STENCIL_NEARBY74 74
#define LSD_STENCIL_EXACT 1000 /* all cells meeting the sqrt(max_sq) ball; accepts d2 <= max_sq */

/* resolution: IVox::Options::resolution_ (0.5, laserMapping.cpp:1061).  log2_lines: the table has
 * 2^log2_lines 128-byte cell lines; keep the load factor <= 0.5 (one line per occupied voxel). */
lsd_status_t lsd_map_create(lsd_map_t** out, float resolution, int log2_lines);
lsd_status_t lsd_map_destroy(lsd_map_t* m);
lsd_status_t lsd_map_clear(lsd_map_t* m);
/* Tile sharding (SURVEY.md §8e): the map keeps only points in x-y tiles (tile_cells voxels wide) this
 * rank owns, plus a halo of reach_cells voxels; queries are answered from the local shard, and lsd_knn_query(_dev) on
 * a sharded map refuses a stencil reaching further than the halo (EXACT: ceil(sqrt(max_sq)/res)+1 voxels). */
lsd_status_t lsd_map_set_shard(lsd_map_t* m, int rank, int world, int tile_cells, int reach_cells);
/* IVox::AddPoints.  Point i is stored with id = id0 + i (ids are what k-NN queries return). */
lsd_status_t lsd_map_insert(lsd_map_t* m, const float* xyzi_host, int n, int32_t id0);
lsd_status_t lsd_map_insert_dev(lsd_map_t* m, const float* xyzi_dev, int n, int32_t id0);
/* IVox::NumValidGrids / NumPoints; n_dropped counts points refused for capacity/range. */
lsd_status_t lsd_map_stats(lsd_map_t* m, uint64_t* n_cells, uint64_t* n_points, uint64_t* n_dropped);
/* KD_TREE::Delete_Point_Boxes (slam/mapping/fastlio/include/ikd-Tree/ikd_Tree.cpp:536-556, Delete_by_range :648-672;
 * how the ikd-Tree path moves its local-map cube, laserMapping.cpp:242-288): deletes every stored point with
 * min <= p < max on all three axes for any of the n_boxes boxes ([n,6] = min xyz, max xyz).  *n_deleted as the
 * reference's return value.  Deleted points can never be returned by a query again; their slots are not reused. */
lsd_status_t lsd_map_delete_boxes(lsd_map_t* m, const float* boxes6_host, int n_boxes, uint64_t* n_deleted);
/* The cudaStream_t every *_dev call of this map is enqueued on (no reference counterpart): lets a
 * caller order its own work after the library's, or time it with CUDA events on the right stream. */
lsd_status_t lsd_map_stream(lsd_map_t* m, void** cuda_stream_out);
/* IVox::GetClosestPoint(pt, out, k, max_sq) for a batch.  k in {1, 5, 20}.  Results per query are
 * sorted ascending by (d2, id); out_idx is -1 padded, out_d2 is -1 padded; out_cnt = #found.
 * fp32 d2 = (dx*dx + dy*dy) + dz*dz without FMA, as ivox3d_node.hpp:11-14 / ikd_Tree.cpp:1374. */
lsd_status_t lsd_knn_query(lsd_map_t* m, const float* q_host, int nq, int k, float max_sq, int stencil,
                           int32_t* out_idx, float* out_d2, int32_t* out_cnt);
lsd_status_t lsd_knn_query_dev(lsd_map_t* m, const float* q_dev, int nq, int k, float max_sq, int stencil,
                               int32_t* out_idx_dev, float* out_d2_dev, int32_t* out_cnt_dev);
/* How the batch is mapped onto the GPU (no reference counterpart; results are bit-identical in every shape):
 * 0 = auto (warp per query below 65 536 queries; from there on the brick pages when lsd_map_enable_bricks was called and
 * the stencil / k are served by them, else thread per query), 1 = warp per query, 2 = thread per query over the voxel
 * lines, 3 = brick pages: the batch is binned by brick, each brick's page (its voxels + a one-voxel halo) is staged into
 * shared memory with one cp.async.bulk (TMA) and answers all its queries from there (csrc/brick.cuh).  Shape 2 serves
 * k in {1, 5} on the fixed stencils; shape 3 k in {1, 5} on CENTER / NEARBY6 / NEARBY18 / NEARBY26; anything else uses
 * shape 1 (shape 3 asked for explicitly on something it does not serve is LSD_ERR_INVALID). */
lsd_status_t lsd_knn_set_shape(lsd_map_t* m, int shape);

/* iVox's capacity and LRU eviction (IVox::Options::capacity_ / max_distance_, ivox3d.h:51-52; AddPoints :231-256: every
 * inserted point moves its voxel to the front of an LRU list, and after every inserted point the voxel at the back is
 * dropped if the map holds more than `capacity` voxels AND the travel distance handed to AddPoints exceeds the distance
 * at which that voxel was created by more than max_distance; the reference runs with 100 000 voxels / 100 m,
 * laserMapping.cpp:1063-1064).  The list order is sequential by nature, so it is replayed on the host from the voxel keys
 * of each insert batch; the evicted voxels' lines are retired on the device (and the table is rebuilt when retired lines
 * crowd it).  Call on an EMPTY map.  lsd_map_set_travel_distance: the `distance` argument of the following AddPoints
 * (lsd_map_insert*) calls; the LIO front-end keeps its own travel_distance (laserMapping.cpp:1289-1291) and needs no
 * call.  Evictions are applied inside the insert calls; lsd_map_evict waits for them and returns how many voxels were
 * evicted so far.  Not on tile-sharded maps, not together with the brick layout; with it on, map_incremental is
 * synchronous (lsd_lio_params::async_map_insert is ignored).  A voxel evicted and re-created inside one batch keeps
 * exactly the points iVox keeps: those the batch added after the voxel's last eviction, whatever their ids. */
lsd_status_t lsd_map_enable_lru(lsd_map_t* m, uint64_t capacity, double max_distance);
lsd_status_t lsd_map_set_travel_distance(lsd_map_t* m, double distance);
/* Test tap: every point the table holds, voxel by voxel (table order), each voxel's points in storage order (its level-0
 * line, then the overflow lines).  Per point: its voxel coordinates (decoded from the key), x, y, z, id, and whether it
 * is a box-delete tombstone (lsd_map_delete_boxes: coordinates set to the quiet NaN 0x7fc00000).  *n_points = the number
 * of stored points, tombstones included; at most `cap` are written (cap = 0 with null arrays asks for the count).
 * Copies the whole table to the host (128 bytes per line): a read-back for tests, not for the per-scan path. */
lsd_status_t lsd_map_dump(lsd_map_t* m, int32_t* voxel3 /*[n,3]*/, float* xyz3 /*[n,3]*/, int32_t* ids /*[n]*/,
                          uint8_t* tombstone /*[n]*/, uint64_t cap, uint64_t* n_points);
lsd_status_t lsd_map_evict(lsd_map_t* m, uint64_t* n_evicted_total);
/* *saturated = 1 when the map refused points since the previous call (probe chain full, > 127 overflow lines in a
 * voxel, coordinates beyond +-2^18 voxels): a map that silently stopped growing degrades odometry, so poll this (the
 * LIO front-end does, and returns LSD_MAP_SATURATED from lsd_lio_scan*). */
lsd_status_t lsd_map_saturated(lsd_map_t* m, int* saturated, uint64_t* n_dropped_total);

/* Brick layout (no reference counterpart: IVox has one layout, a hash of per-voxel point lists, ivox3d.h:31-112; this is
 * the same content arranged for batched queries).  After this call every point the map accepts is ALSO stored in the
 * 4608-byte page of each 8 x 8 x 4-voxel brick whose one-voxel halo contains it (points already in the map are copied
 * over), lsd_map_delete_boxes tombstones the replicas too, and lsd_knn_query* may use shape 3.  The directory has
 * 2^log2_bricks slots (memory: 4.6 KB per slot); size it for <= 0.5 load: a 10 M-point outdoor map at 0.5 m needs about
 * 170 k pages.  Not available on tile-sharded maps.  lsd_map_brick_stats: pages in use, point replicas stored, replicas
 * dropped for capacity (must stay 0 for shape 3 to be exact). */
lsd_status_t lsd_map_enable_bricks(lsd_map_t* m, int log2_bricks);
lsd_status_t lsd_map_brick_stats(lsd_map_t* m, uint64_t* n_pages, uint64_t* n_replicas, uint64_t* n_dropped);

/* ------------------------------------------------------------------------------------------
 * Voxel-grid downsample — replaces pcl::VoxelGrid<PointXYZINormal>::filter as called at
 * laserMapping.cpp:1206-1207 (leaf 0.5) and hdl_localization_nodelet.cpp:333-344.
 * Output: one centroid (all 4 channels) per occupied leaf, ascending leaf index like PCL.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_voxelgrid lsd_voxelgrid_t;
lsd_status_t lsd_voxelgrid_create(lsd_voxelgrid_t** out, int max_points, int log2_max_cells);
lsd_status_t lsd_voxelgrid_destroy(lsd_voxelgrid_t* g);
/* out_host must hold n points; *m receives the output count. */
lsd_status_t lsd_voxelgrid_filter(lsd_voxelgrid_t* g, const float* in_host, int n, float leaf, float* out_host, int* m);
lsd_status_t lsd_voxelgrid_filter_dev(lsd_voxelgrid_t* g, const float* in_dev, int n, float leaf, float* out_dev,
                                      int* m_dev);

/* ------------------------------------------------------------------------------------------
 * LIO front-end — replaces the per-scan body of fastlio_main (laserMapping.cpp:1126-1387):
 * VoxelGrid -> iterated ESKF update (esekf::update_iterated_dyn_share_modified,
 * IKFoM_toolkit/esekfom/esekfom.hpp:1619-1931) with h_share_model_geometric
 * (laserMapping.cpp:813-982) -> map_incremental (laserMapping.cpp:523-576).
 *
 * State vector (26 doubles), state_ikfom of use-ikfom.hpp:12-21 with quaternions as (x,y,z,w):
 *   pos[3] rot[4] offset_R_L_I[4] offset_T_L_I[3] vel[3] bg[3] ba[3] grav[3]
 * Covariance: 23x23 row-major doubles (DOF order pos, rot, offset_R, offset_T, vel, bg, ba, grav2).
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_lio lsd_lio_t;

typedef struct lsd_lio_params {
  int max_points;            /* scratch capacity; reference static cap 100000, laserMapping.cpp:86   */
  int max_scan_points;       /* raw scan capacity for lsd_lio_scan (pre-downsample)                 */
  float filter_size_surf;    /* 0.5, laserMapping.cpp:1027                                          */
  float filter_size_map;     /* 0.5, laserMapping.cpp:1028                                          */
  float ivox_resolution;     /* 0.5, laserMapping.cpp:1061                                          */
  int ivox_nearby;           /* LSD_STENCIL_*; reference: NEARBY74 first second, then NEARBY18      */
  int map_log2_lines;        /* hash table size                                                     */
  int max_iterations;        /* NUM_MAX_ITERATIONS = 4, laserMapping.cpp:1026                       */
  double laser_point_cov;    /* LASER_POINT_COV = 0.001, laserMapping.cpp:71                        */
  double converge_eps;       /* 0.001, laserMapping.cpp:1114-1116                                   */
  int degenerate_detect_en;  /* laserMapping.cpp:83                                                 */
  int knn_mode_exact;        /* 0: iVox stencil (live path), 1: exact k-NN (ikd-Tree path)          */
  int eskf_literal;          /* 1: evaluate the Kalman gain with the reference's two dense 23x23
                                inversions (esekfom.hpp:1756-1789); 0 (default): the algebraically
                                identical Schur-complement form (two 6x6 inverses), ~2x faster on
                                the host and equally accurate (DESIGN.md "Host ESKF")             */
  int async_map_insert;      /* 1: lsd_lio_scan returns as soon as the pose is final; map_incremental
                                completes in the background on the handle's stream (the next call is
                                ordered after it).  info->gpu_ms / n_added then describe the PREVIOUS
                                scan; lsd_lio_sync() drains.  0 (default): fully synchronous.          */
} lsd_lio_params_t;

typedef struct lsd_lio_info {
  int n_down;       /* feats_down_size                                   */
  int iterations;   /* h-model evaluations run                            */
  int n_eff;        /* effct_feat_num of the last evaluation              */
  int degenerate;   /* is_degenerate of the last evaluation               */
  int n_added;      /* points inserted by map_incremental                 */
  int converged;    /* the update returned through the t > 1 exit         */
  double res_mean;  /* res_mean_last                                      */
  double gpu_ms;    /* device time of this scan (CUDA events)             */
  int kernel_launches;
} lsd_lio_info_t;

void lsd_lio_default_params(lsd_lio_params_t* p);
lsd_status_t lsd_lio_create(lsd_lio_t** out, const lsd_lio_params_t* p);
lsd_status_t lsd_lio_destroy(lsd_lio_t* l);
lsd_map_t* lsd_lio_map(lsd_lio_t* l);
lsd_status_t lsd_lio_set_nearby(lsd_lio_t* l, int stencil); /* IVox::SetNearByType, laserMapping.cpp:1241-1243 */
lsd_status_t lsd_lio_set_ekf_inited(lsd_lio_t* l, int flag);
/* The reference's stale Nearest_Points rows.  Nearest_Points is a file-scope vector<PointVector> that is only resize()d
 * per scan (laserMapping.cpp:1273), and IVox::GetClosestPoint returns BEFORE clearing its output when no map point is in
 * range (ivox3d.h:155-157): a scan point with nothing near it keeps the neighbours row i held the last time a search
 * found any (an earlier iteration or an earlier scan), is plane-fitted and gated on those, and map_incremental reads
 * them too.  flag != 0 reproduces that (iVox stencils on a single-GPU handle; the exact / ikd-Tree search clears its
 * output); 0 (default this round, see DESIGN.md section 4) treats such a point as having no neighbours.  Either call
 * empties the rows. */
lsd_status_t lsd_lio_set_stale_rows(lsd_lio_t* l, int flag);
/* The reference's neighbour ORDER.  IVox::GetClosestPoint returns its (up to) five neighbours in the order two std::nth_element
 * calls leave them in (ivox3d.h:159-164; one more per voxel with over five points in range, ivox3d_node.hpp:118-123), and
 * esti_plane's fp32 least-squares solve (common_lib.h:251) depends on the order of its rows: on a map a kilometre from the
 * origin the row order alone moves plane distances by over 1e-4 m.  flag != 0: Nearest_Points rows hold the reference's
 * neighbours in the reference's order (libstdc++'s introselect replayed on the candidate sequence the reference builds), which
 * together with esti_plane in Eigen's summation order makes the per-scan posterior equal to laserMapping.cpp's to rounding of
 * the double-precision sums — the DEFAULT; 0: ascending (d2, id), 9 % more scans/s, posterior ~4e-5 m from the reference's.
 * iVox stencils only (the exact / ikd-Tree search returns sorted neighbours).  LSD_REF_ORDER=0 in the environment turns it off
 * at lsd_lio_create.
 * lsd_lio_reference_order_fallbacks: scan points since creation whose stencil held more than 256 in-range map points
 * (those are answered in (d2, id) order).  A registered scan takes 2 n ids instead of n while the switch is on (ids then grow
 * in the reference's insertion order: every PointToAdd of a scan before every PointNoNeedDownsample). */
lsd_status_t lsd_lio_set_reference_order(lsd_lio_t* l, int flag);
lsd_status_t lsd_lio_reference_order_fallbacks(lsd_lio_t* l, unsigned* count);
/* Test entry for the above: libstdc++'s std::nth_element(first, nth, last) (bits/stl_algo.h __introselect) as the search kernel
 * replays it, on n <= 256 non-negative distances (host pointers).  perm_out[p] = index of the element at position p afterwards;
 * path_out (optional): 1 = warp-cooperative replay, 2 = it left at introselect's depth limit and the serial replay took over,
 * 3 = serial replay (n > 32). */
lsd_status_t lsd_debug_nth_element(const float* dist_host, int n, int first, int nth, int last, int* perm_out_host, int* path_out_host);
/* Test entry: the LIO search's plane fit (esti_plane, common_lib.h:236-268) alone, one device thread per set.  pts5_host
 * [n,5,3] (host), thr the residual threshold; pabcd_out [n,4] the plane (a, b, c, d), ok_out [n] 1 where every point is
 * within thr of it. */
lsd_status_t lsd_debug_esti_plane(const float* pts5_host, int n, float thr, float* pabcd_out, int* ok_out);
/* Shape of the per-scan neighbour search (no reference counterpart): 0 or 1 = one warp per scan point (the only shape;
 * the flat shapes of round 1 were retired). */
lsd_status_t lsd_lio_set_knn_shape(lsd_lio_t* l, int shape);
/* Programmatic dependent launch for the per-scan kernel chain (no reference counterpart; results are bit-identical either
 * way): flag != 0 launches the voxel-grid, search, h-model and map_incremental kernels with the programmatic stream
 * serialization attribute, so that each kernel's blocks are resident and parked in griddepcontrol.wait when its
 * predecessor drains (csrc/lsd_common.cuh).  Default 0, or 1 when LSD_PDL=1 is in the environment at lsd_lio_create;
 * ignored on a tile-sharded handle. */
lsd_status_t lsd_lio_set_pdl(lsd_lio_t* l, int flag);
/* Id given to the next point map_incremental inserts (ids of points inserted through
 * lsd_map_insert(lsd_lio_map(l), ...) are the caller's). */
lsd_status_t lsd_lio_set_next_id(lsd_lio_t* l, int32_t id); /* flg_EKF_inited, laserMapping.cpp:1196 */

/* Per-kernel CUDA-event timing for the roofline report (adds a sync per launch: never enable it in a
 * throughput measurement).  ms4/cnt4: [0] h-model with k-NN search, [1] h-model reusing neighbours,
 * [2] voxel grid (7 kernels), [3] map_incremental. */
/* Tile-sharded LIO across the GPUs of one box (no reference counterpart: the reference is single-GPU /
 * CPU, SURVEY.md §2.6).  Every rank runs the same lsd_lio_* calls in lock-step on the same scans; a rank
 * resolves the queries whose home voxel it owns, the 30-double normal equations are all-reduced inside
 * the reduction kernel through peer memory (NVLink stores into every rank's inbox, rank-ordered fold),
 * and map_incremental's decisions are exchanged the same way so halo copies stay consistent.
 *   1. every rank: lsd_lio_shard_export(l, rank, world, tile_cells, reach_cells, blob)   (<= 8 ranks)
 *   2. all-gather the LSD_SHARD_BLOB_BYTES blobs (torch.distributed / MPI / a pipe)
 *   3. every rank: lsd_lio_shard_connect(l, blobs[world])
 * reach_cells: 1 for NEARBY6/18/26, 2 for NEARBY74, ceil(sqrt(5)/res)+1 for the exact search (6 at res 0.5); tile_cells
 * must exceed 2 * reach_cells.  Enforced: with world > 1, lsd_lio_shard_export refuses (LSD_ERR_INVALID) a reach_cells
 * below what the handle's search needs, and lsd_lio_set_nearby refuses a stencil the exported halo cannot serve —
 * a narrower halo would not fail, it would silently drop neighbours of queries near a tile border. */
#define LSD_SHARD_BLOB_BYTES 192
lsd_status_t lsd_lio_shard_export(lsd_lio_t* l, int rank, int world, int tile_cells, int reach_cells, unsigned char* blob_out);
lsd_status_t lsd_lio_shard_connect(lsd_lio_t* l, const unsigned char* blobs);
/* Tile-sharded handles: mean time (us) one h-model evaluation spent in the in-kernel exchange — the peer-memory stores plus
 * waiting for the slowest peer's partial sums (clock64 around it, nominal SM clock) — over the evaluations since the
 * last call. */
lsd_status_t lsd_lio_shard_exchange_stats(lsd_lio_t* l, double* mean_us, long long* evaluations);
/* Wait for everything queued on the handle; returns device time / insert count of the last scan. */
lsd_status_t lsd_lio_sync(lsd_lio_t* l, double* gpu_ms_last, int* n_added_last);
lsd_status_t lsd_lio_set_profile(lsd_lio_t* l, int on);
lsd_status_t lsd_lio_get_profile(lsd_lio_t* l, double* ms4, long long* cnt4);

/* Load the undistorted scan (feats_undistort) and, if `downsample`, run the 0.5 m VoxelGrid
 * (laserMapping.cpp:1206-1207).  Returns the downsampled size in *n_down. */
lsd_status_t lsd_lio_load_scan(lsd_lio_t* l, const float* scan_host, int n, int downsample, int* n_down);
lsd_status_t lsd_lio_load_scan_dev(lsd_lio_t* l, const float* scan_dev, int n, int downsample, int* n_down);
/* Copy back the downsampled scan (feats_down_body), [n_down,4]. */
lsd_status_t lsd_lio_get_down(lsd_lio_t* l, float* out_host, int cap, int* n_down);

/* One evaluation of h_share_model_geometric on the loaded scan at `state`; search != 0 redoes the
 * k-NN (ekfom_data.converge).  HTH[36]: the non-zero 6x6 block of h_x^T h_x; HTh[6] = h_x^T h.
 * Returns LSD_NO_EFFECTIVE_POINTS when n_eff < 1. */
lsd_status_t lsd_lio_linearize(lsd_lio_t* l, const double* state26, int search, double* HTH36, double* HTh6,
                               double* res_sum, int* n_eff, int* degenerate);
/* Debug/parity taps after lsd_lio_linearize: per downsampled point neighbours, plane and flags. */
lsd_status_t lsd_lio_get_matches(lsd_lio_t* l, int32_t* near_idx /*[n,5]*/, float* near_xyz /*[n,5,3]*/,
                                 int32_t* near_cnt /*[n]*/, uint8_t* selected /*[n]*/, float* plane /*[n,4]*/,
                                 float* world /*[n,4]*/);
/* esekf::update_iterated_dyn_share_modified on the loaded scan. */
lsd_status_t lsd_lio_update(lsd_lio_t* l, double* state26_inout, double* P529_inout, lsd_lio_info_t* info);
/* map_incremental at `state` using the neighbour lists of the last search. */
lsd_status_t lsd_lio_map_incremental(lsd_lio_t* l, const double* state26, int* n_added);
/* Test tap after a map_incremental: the decision per downsampled point (0 = not added, 1 = PointToAdd, 2 =
 * PointNoNeedDownsample; laserMapping.cpp:523-576) and the travel distance the LIO front-end handed the map's LRU.
 * With lsd_lio_get_matches' `world` this is enough to restate the scan's two AddPoints calls (laserMapping.cpp:571-572).
 * Writes at most `cap` flags; *n = the number of downsampled points. */
lsd_status_t lsd_lio_get_map_flags(lsd_lio_t* l, uint8_t* flags, int cap, int* n, double* travel_distance);
/* The whole per-scan pass: load (+downsample) -> [seed map | update -> map_incremental]. */
lsd_status_t lsd_lio_scan(lsd_lio_t* l, const float* scan_host, int n, double* state26_inout, double* P529_inout,
                          lsd_lio_info_t* info);
lsd_status_t lsd_lio_scan_dev(lsd_lio_t* l, const float* scan_dev, int n, double* state26_inout,
                              double* P529_inout, lsd_lio_info_t* info);
/* Double-buffered ingest (no reference counterpart: the reference copies nothing).  Starts the host->device copy
 * of the NEXT scan on a copy stream and returns at once; a following lsd_lio_scan with the same (pointer, n)
 * uses the staged copy instead of uploading again, so the PCIe transfer of scan k+1 overlaps the registration
 * of scan k.  The host buffer must stay unchanged (and, to overlap, pinned) until that lsd_lio_scan returns. */
lsd_status_t lsd_lio_prefetch(lsd_lio_t* l, const float* scan_host, int n);
/* Pipelined voxel grid (no reference counterpart; bit-identical results).  The downsample of a scan depends on nothing the
 * previous scan computes, so with flag != 0 a prefetched scan is also voxel-grid filtered ahead — on the copy stream, behind
 * its copy, while the previous scan iterates — and the lsd_lio_scan that adopts it starts at its first neighbour search.
 * Default 0, or 1 when LSD_PIPELINE_VG=1 is in the environment at lsd_lio_create; ignored on a tile-sharded handle. */
lsd_status_t lsd_lio_set_pipeline(lsd_lio_t* l, int flag);
/* How many scans were downsampled ahead, and how many of those a later lsd_lio_scan adopted (either pointer may be NULL). */
lsd_status_t lsd_lio_pipeline_stats(lsd_lio_t* l, long long* issued, long long* adopted);
/* The same announcement for a device-resident scan (the pointer later passed to lsd_lio_scan_dev, unchanged until then):
 * nothing to copy, so this only does something when the pipelined voxel grid is on. */
lsd_status_t lsd_lio_prefetch_dev(lsd_lio_t* l, const float* scan_dev, int n);

/* ------------------------------------------------------------------------------------------
 * Scan matcher — replaces what select_registration_method() hands out
 * (slam/backend/hdl_graph_slam/include/hdl_graph_slam/registrations.hpp:15-16, registrations.cpp:29-155):
 * fast_gicp::NDTCuda ("NDT_CUDA": P2D, DIRECT7, res 1.0, 64 iters, eps 0.01 / 0.1 deg) and
 * fast_gicp::FastGICP ("FAST_GICP": k = 20, max-corr 2.0 m), both driven by
 * fast_gicp::LsqRegistration's Levenberg-Marquardt loop (lsq_registration_impl.hpp:71-208), plus
 * pcl::Registration::getFitnessScore.  Call protocol mirrors pcl::Registration:
 *   setInputTarget -> lsd_reg_set_target, setInputSource -> lsd_reg_set_source,
 *   align(out, guess) -> lsd_reg_align, hasConverged / getFinalTransformation -> its outputs,
 *   getFitnessScore(max_range) -> lsd_reg_fitness, setMaxCorrespondenceDistance -> same name.
 * Transforms are 4x4 row-major.  A handle is confined to one thread at a time; set_target on one handle may
 * run concurrently with align on another (the localisation ping-pong, hdl_localization_nodelet.cpp:291-307).
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_reg lsd_reg_t;
#define LSD_REG_NDT_P2D 0
#define LSD_REG_GICP 1
#define LSD_REG_VGICP 2     /* fast_gicp::FastVGICP ("FAST_VGICP", registrations.cpp:56-66) */

typedef struct lsd_reg_params {
  int kind;                       /* LSD_REG_NDT_P2D | LSD_REG_GICP | LSD_REG_VGICP                        */
  double resolution;              /* NDT voxel size (1.0, registrations.cpp:106)                          */
  int ndt_neighbors;              /* 1 | 7 | 27 = DIRECT1 / DIRECT7 / DIRECT27 (ndt_cuda.cu:35-69)        */
  int max_iterations;             /* 64                                                                   */
  double transformation_epsilon;  /* 0.01                                                                 */
  double rotation_epsilon_deg;    /* NDT 0.1; LsqRegistration default 1e-2 (compared against degrees)     */
  int lm_max_iterations;          /* 10  (lsq_registration_impl.hpp:30)                                   */
  double lm_init_lambda_factor;   /* 1e-9 (lsq_registration_impl.hpp:31)                                  */
  int64_t max_process_time_us;    /* soft timeout, hard stop at 1.5x (lsq_registration_impl.hpp:94-104)   */
  int k_correspondences;          /* GICP covariance neighbourhood, 20 (<= 20)                            */
  double max_corr_dist;           /* GICP max correspondence distance, 2.0 m                              */
  double normal_search_sq;        /* GICP: squared radius of the FAST grid search for the k-NN (25 m^2); points with
                                     fewer than k neighbours inside it get the true k-NN by an exact scan of the cloud,
                                     so the result is nearestKSearch's (fast_gicp_impl.hpp:259) whatever this is        */
  double map_resolution;          /* voxel size of the exact-NN index (0.5 m)                             */
  int map_log2_lines;             /* hash table size, 0 = derive from the cloud size                      */
} lsd_reg_params_t;

/* Tile-sharded matcher (SURVEY.md section 8e, row C3: "NDT localisation: the 50 M-point map voxelised per tile on the owner
 * GPU, all-reduce of [H, b, err] per LM trial").  No reference counterpart (the reference's NDTCuda is single-GPU,
 * ndt_cuda.cu:115-178).  NDT_P2D only: after export / all-gather / connect (the hand-shake of lsd_lio_shard_*, same
 * blob size), lsd_reg_set_target* keeps only the voxels of the x-y tiles (tile_cells NDT voxels wide) this rank owns —
 * the caller may pass the whole cloud or just the points of its own tiles — every rank sets the SAME source and runs
 * the SAME lsd_reg_align / lsd_reg_cost calls in lockstep; the 28 sums of every cost evaluation are all-reduced inside
 * the reduction kernel through peer memory (rank-ordered fold: bit-identical on every rank), so all ranks return the same
 * pose.  lsd_reg_fitness is not available on a sharded handle. */
lsd_status_t lsd_reg_shard_export(lsd_reg_t* r, int rank, int world, int tile_cells, unsigned char* blob_out);
lsd_status_t lsd_reg_shard_connect(lsd_reg_t* r, const unsigned char* blobs);


void lsd_reg_default_params(lsd_reg_params_t* p, int kind);
lsd_status_t lsd_reg_create(lsd_reg_t** out, const lsd_reg_params_t* p);
lsd_status_t lsd_reg_destroy(lsd_reg_t* r);
lsd_status_t lsd_reg_set_target(lsd_reg_t* r, const float* pts_host, int n);      /* [n,4] */
lsd_status_t lsd_reg_set_target_dev(lsd_reg_t* r, const float* pts_dev, int n);
lsd_status_t lsd_reg_set_source(lsd_reg_t* r, const float* pts_host, int n);
lsd_status_t lsd_reg_set_source_dev(lsd_reg_t* r, const float* pts_dev, int n);
lsd_status_t lsd_reg_set_max_correspondence_distance(lsd_reg_t* r, double d);
/* align(): guess/out are float32[16] like Eigen::Matrix4f; *converged = hasConverged(). */
lsd_status_t lsd_reg_align(lsd_reg_t* r, const float* guess16, float* out16, int* converged, int* iterations);
/* Diagnostics of the last lsd_reg_align (no reference counterpart beyond lm_debug_print_, lsq_registration_impl.hpp:176-183):
 * per outer LM iteration 4 doubles = (|translation|_inf of the accepted step [m], its rotation angle [deg] — the two numbers
 * is_converged compares with transformation_epsilon / rotation_epsilon, :112-121 — the cost at the linearisation, lambda).
 * out may be NULL to learn *n_iters. */
lsd_status_t lsd_reg_iteration_log(lsd_reg_t* r, double* out4_per_iter, int cap_iters, int* n_iters);
lsd_status_t lsd_reg_get_final(lsd_reg_t* r, double* T16, double* H36);           /* double pose, getFinalHessian */
/* getFitnessScore(max_range) at T16 (NULL = the final transformation).  NB PCL compares the SQUARED
 * nearest-neighbour distance with max_range.  The nearest neighbour is exact at any range: past the point map's grid
 * search (64 map voxels) and on a target whose point map refused points, it comes from a scan of the whole target. */
lsd_status_t lsd_reg_fitness(lsd_reg_t* r, const double* T16_or_null, double max_range, double* score);
/* One cost evaluation (parity tap): update != 0 = linearize(T) (correspondences refreshed), else
 * compute_error(T).  H36/b6 may be NULL. */
lsd_status_t lsd_reg_cost(lsd_reg_t* r, const double* T16, int update, double* H36, double* b6, double* err, int* n_corr);
/* Parity tap: the correspondences of the last linearisation.  GICP: [n_src] target point index or -1
 * (correspondences_, fast_gicp_impl.hpp:119-157); NDT / VGICP: [neighbors, n_src] voxel-table slot or -1. */
lsd_status_t lsd_reg_get_correspondences(lsd_reg_t* r, int32_t* corr_host, int cap, int* n);
lsd_status_t lsd_reg_stats(lsd_reg_t* r, int* n_voxels, long long* launches);
/* Read-back taps of the target / source build (GICP and VGICP handles).
 * lsd_reg_get_covariances: the k-NN covariance of every point of the target (which = 1) or source (which = 0) as
 * [n, 4] doubles = (smallest-eigenvalue direction, neighbour count) — what calculate_covariances
 * (fast_gicp_impl.hpp:244-303) reduces to under PLANE regularisation.  out must hold 4 * n doubles.
 * lsd_reg_get_voxels: every occupied line of the current target voxel table, in table order, *n_out = their number (at
 * most cap are written; any output may be NULL when cap = 0).  coord [cap, 3] = voxel coordinates decoded from the key,
 * count = points in the voxel, mean [cap, 3].  VGICP (GaussianVoxelMap::create_voxelmap + AdditiveGaussianVoxel::finalize,
 * fast_vgicp_voxel.hpp:108-182): second [cap, 6] = the mean of the points' I - 0.999 n n^T (xx xy xz yy yz zz).  NDT
 * (gaussian_voxelmap.cu:181-202): second[0..2] = the stored smallest-eigenvalue direction, widened from float,
 * second[3..5] = 0.  LSD_ERR_INVALID on a GICP handle (no voxel table) or before a target is set. */
lsd_status_t lsd_reg_get_covariances(lsd_reg_t* r, int which, double* out);
lsd_status_t lsd_reg_get_voxels(lsd_reg_t* r, int cap, int* coord, int* count, double* mean, double* second, int* n_out);

/* ------------------------------------------------------------------------------------------
 * Loop-closure detector — replaces hdl_graph_slam::LoopDetector
 * (slam/backend/hdl_graph_slam/include/hdl_graph_slam/loop_detector.hpp:33-231, called from
 * hdl_graph_slam_nodelet.cpp:613) and the fitness part of InformationMatrixCalculator
 * (information_matrix_calculator.cpp:25-47,71-102).  Key-frame clouds (sensor frame) are uploaded once into a
 * device pool and addressed by slot.  The coarse stage (NDT_CUDA of every candidate against the new key frame,
 * :148-191) runs all candidates together: one batched cost launch per Levenberg-Marquardt round for the whole
 * candidate set, each candidate bit-identical to a separate lsd_reg NDT handle on the same pair.  The refinement
 * (FAST_GICP, max-corr 0.5 m, :193-219) runs on the one best pair through the lsd_reg GICP code.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_loop lsd_loop_t;
typedef struct lsd_loop_params {
  double distance_thresh;                 /* 15.0 m, x-y distance of the graph estimates (loop_detector.hpp:43,129-133) */
  double accum_distance_thresh;           /* 25.0 m travelled between candidate and new key frame (:44,119-121)        */
  double distance_from_last_edge_thresh;  /* 15.0 m travelled since the last accepted loop (:45,108-110)              */
  double distance_new_keyframe_thresh;    /* 2.0 m between the new key frames examined in one detect (:46,78-80)      */
  double distance_keyframe_thresh;        /* 2.0 m between accepted candidates (:47,123-125)                          */
  double fitness_score_max_range;         /* 25.0, SQUARED distance as PCL compares it (:49,180,206)                   */
  double fitness_score_thresh;            /* 1.5 (:50; the coarse gate is 2x this, :193)                              */
  lsd_reg_params_t coarse;                /* lsd_reg_default_params(LSD_REG_NDT_P2D): "NDT_CUDA", registrations.cpp:107-118;
                                             max_process_time_us must be 0 (the reference sets no timeout)             */
  lsd_reg_params_t accurate;              /* LSD_REG_GICP with max_corr_dist = 0.5 (loop_detector.hpp:58-59)           */
} lsd_loop_params_t;

typedef struct lsd_loop_result {
  int32_t key1, key2;          /* new key frame slot, matched candidate slot (Loop::key1 / key2)                     */
  float relpose16[16];         /* registration_accurate->getFinalTransformation(), row-major (:216)                  */
  double coarse_score, score;  /* best NDT getFitnessScore (:180), final GICP getFitnessScore (:206)                 */
  double information36[36];    /* calc_information_matrix(key1 cloud, key2 cloud, relpose), row-major               */
  int32_t n_candidates;        /* candidates the coarse stage matched                                                 */
} lsd_loop_result_t;

/* What detect decided for each new key frame it was given (no reference counterpart beyond its LOG_INFO lines). */
#define LSD_LOOP_SKIPPED 0         /* closer than distance_new_keyframe_thresh to the previous one examined (:78-80) */
#define LSD_LOOP_NO_CANDIDATES 1   /* find_candidates returned nothing (:150-152)                                    */
#define LSD_LOOP_COARSE_REJECT 2   /* best NDT score above 2 * fitness_score_thresh, or nothing converged (:193-196) */
#define LSD_LOOP_GICP_DIVERGED 3   /* the refinement did not converge (:202-205)                                     */
#define LSD_LOOP_GICP_REJECT 4     /* the refined score is above fitness_score_thresh (:206-210)                     */
#define LSD_LOOP_FOUND 5
typedef struct lsd_loop_report {
  int32_t new_slot, decision, n_candidates, best_slot;  /* best_slot: the coarse stage's choice, -1 = none   */
  double best_score;                                    /* its NDT score (DBL_MAX when nothing converged)   */
} lsd_loop_report_t;

void lsd_loop_default_params(lsd_loop_params_t* p);
lsd_status_t lsd_loop_create(lsd_loop_t** out, const lsd_loop_params_t* p);
lsd_status_t lsd_loop_destroy(lsd_loop_t* h);
/* KeyFrame (keyframe.hpp:21-41): its cloud (sensor frame, [n,4]) is uploaded once and kept on the device;
 * accum_distance as KeyFrame::accum_distance.  *slot = 0, 1, 2, ... in call order. */
lsd_status_t lsd_loop_add_keyframe(lsd_loop_t* h, const float* xyzi_host, int n, double accum_distance, int32_t* slot);
/* LoopDetector::detect (:69-91).  poses16 = the current graph estimate of EVERY slot ([n_slots,16], double, row-major,
 * node->estimate()); keyframes / new_keyframes = slots in the order of the reference's vector / deque.  Writes up to
 * cap loops; *n_loops = loops found (may exceed cap).  last_edge_accum_distance persists across calls (:60,216). */
lsd_status_t lsd_loop_detect(lsd_loop_t* h, const double* poses16, const int32_t* keyframes, int n_kf,
                             const int32_t* new_keyframes, int n_new, lsd_loop_result_t* out, int cap, int* n_loops);
/* Per new key frame of the last lsd_loop_detect, in order: what was decided (LSD_LOOP_*).  out may be NULL. */
lsd_status_t lsd_loop_last_reports(lsd_loop_t* h, lsd_loop_report_t* out, int cap, int* n);
/* last_edge_accum_distance (:216) of the handle: read (get != 0) or set. */
lsd_status_t lsd_loop_last_edge(lsd_loop_t* h, double* value, int get);
/* find_candidates (:106-140) and the initial guess of each candidate (:165-173: both rotations normalised through a
 * quaternion, new^-1 * candidate in double, cast to float, element (2,3) zeroed; returned as double).  Pure host: works
 * without a device.  accum = KeyFrame::accum_distance of every slot.  *n_cand = candidates found (may exceed cap). */
lsd_status_t lsd_loop_find_candidates(const lsd_loop_params_t* p, double last_edge_accum_distance, const double* poses16,
                                      const double* accum, const int32_t* keyframes, int n_kf, int32_t new_slot,
                                      int32_t* cand_out, double* guesses16_out, int cap, int* n_cand);
/* Parity tap: the coarse stage alone (:158-191 without the selection) for an explicit candidate list against target_slot.
 * Per candidate: final NDT pose (double [n,16]), converged, iterations (hasConverged / the LM iteration count of
 * lsd_reg_align), getFitnessScore(fitness_score_max_range) at that pose.  Any output may be NULL.  *launches / *rounds:
 * kernel launches and host round trips (one batched cost evaluation each) the call used. */
lsd_status_t lsd_loop_match(lsd_loop_t* h, int32_t target_slot, const int32_t* cand, const double* guesses16, int n,
                            double* final16, int32_t* converged, int32_t* iterations, double* fitness, long long* launches,
                            int* rounds);
/* The LM iteration log of candidate i of the last lsd_loop_match, same layout as lsd_reg_iteration_log. */
lsd_status_t lsd_loop_iteration_log(lsd_loop_t* h, int i, double* out4_per_iter, int cap_iters, int* n_iters);
/* calc_fitness_score(target cloud, source cloud, T, max_range) (information_matrix_calculator.cpp:71-102): mean squared
 * distance of every transformed source point to its nearest target point, however far (max_range = DBL_MAX counts them
 * all).  T16 is applied in float, as pcl::transformPointCloud does. */
lsd_status_t lsd_loop_fitness(lsd_loop_t* h, int32_t target_slot, int32_t source_slot, const float* T16, double max_range,
                              double* score, int* n_counted);
/* InformationMatrixCalculator::calc_information_matrix(fitness_score) (:49-62): identity / w_x (translation), / w_q
 * (rotation), w_* = weight() stored in float.  Pure host. */
void lsd_loop_information_matrix(double fitness_score, double* information36);

/* ------------------------------------------------------------------------------------------
 * Global alignment search — replaces the closure search of global_alignment
 * (slam/localization/include/global_alignment.hpp:200-258, called from MapLoader::mergeMapSLAM,
 * slam/localization/src/map_loader.cpp:82-169, when either map has no GNSS origin).  Key-frame clouds (sensor frame) are
 * uploaded once into a device pool, addressed by slot and marked as reference (the loaded map) or new (the map being
 * merged); each reference key frame's ScanContext (offset (0, 0), keyframe.cpp:165-167) enters a database in slot order, so
 * the database index is the reference index.  A reference key frame's point map, k = 20 covariances and VGICP voxel table
 * are built on its first use as a target and kept; a new key frame's covariances once.  lsd_galign_search does, for all new
 * key frames given: nine-offset descriptors (:209-214), detectCandidateMatch merged per reference (:215-227), FAST_VGICP of
 * every (new, reference) pair from yaw2matrix(-sc_yaw) (:231-244) with the Levenberg-Marquardt loops of all pairs
 * advanced together (one batched cost launch per round), getFitnessScore(25) of all pairs in one launch (:249), and the
 * gate converged && score < 1.5 (:245-253).  Each pair is bit-identical to the single-pair kernels on the same tables.
 * The PCM matrix, max-clique and estimate_transform (:261-300) stay with the caller.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_galign lsd_galign_t;
typedef struct lsd_galign_params {
  lsd_reg_params_t reg;             /* lsd_reg_default_params(LSD_REG_VGICP): select_registration_method("FAST_VGICP")
                                       (registrations.cpp:56-66: res 1.0, eps 0.1 m / 0.1 deg, 64 iterations, k = 20),
                                       max_process_time_us must be 0                                                     */
  double sc_dist_thres;             /* 0.30, SC_DIST_THRES (global_alignment.hpp:31)                                    */
  double icp_score_thres;           /* 1.5, ICP_SCORE_THRES (:32); a closure needs score < this                        */
  double fitness_score_max_range;   /* 25, FITNESS_SCORE_MAX (:34), SQUARED distance as PCL compares it                */
  int64_t max_batch_points;         /* pair budget of one batch: sum over its pairs of new-cloud points x ndt_neighbors
                                       (4 + 48 bytes each for correspondences and Mahalanobis matrices).  A search splits
                                       into batches of whole new key frames; results do not depend on the split.  2^24 */
  int sc_db_capacity;               /* reference key frames the ScanContext database holds (4096)                       */
} lsd_galign_params_t;

typedef struct lsd_galign_closure {
  int32_t ref_slot, new_slot;  /* Closures(key1 = reference key frame, key2 = new key frame) (:251)                 */
  float relpose16[16];         /* registration->getFinalTransformation(), row-major: new key frame -> reference   */
  double score;                /* getFitnessScore(fitness_score_max_range) (:249)                                 */
  float sc_dist, sc_yaw;       /* the merged SCMatch: distance and yaw (rad) of the ScanContext match             */
} lsd_galign_closure_t;

typedef struct lsd_galign_match {
  int32_t new_slot, ref_slot;
  float sc_dist, sc_yaw;
  int32_t converged, iterations;
  double score;                /* getFitnessScore at the final pose (computed for every pair)                      */
  int32_t accepted;            /* converged && score < icp_score_thres                                            */
} lsd_galign_match_t;

void lsd_galign_default_params(lsd_galign_params_t* p);
lsd_status_t lsd_galign_create(lsd_galign_t** out, const lsd_galign_params_t* p);
lsd_status_t lsd_galign_destroy(lsd_galign_t* h);
/* KeyFrame::mPoints ([n,4], sensor frame) uploaded once; reference != 0 adds it to the reference map (and its
 * ScanContext to the database), else to the new map.  *slot = 0, 1, 2, ... in call order. */
lsd_status_t lsd_galign_add_keyframe(lsd_galign_t* h, const float* xyzi_host, int n, int reference, int32_t* slot);
/* The search of :206-258 for the new key frames new_slots (in that order).  Writes up to cap closures, ordered by new key
 * frame, then ascending reference index; *n_closures = closures found (may exceed cap). */
lsd_status_t lsd_galign_search(lsd_galign_t* h, const int32_t* new_slots, int n_new, lsd_galign_closure_t* out, int cap,
                               int* n_closures);
/* Sets max_batch_points (> 0) for the following searches: the memory a search may hold for correspondences and Mahalanobis
 * matrices at once.  Results do not depend on it. */
lsd_status_t lsd_galign_set_max_batch_points(lsd_galign_t* h, int64_t max_batch_points);
/* Every pair the last lsd_galign_search aligned, in its order.  out may be NULL. */
lsd_status_t lsd_galign_last_matches(lsd_galign_t* h, lsd_galign_match_t* out, int cap, int* n);
/* Work of the last lsd_galign_search: kernel launches of the matching (tables, cost rounds, fitness), host round trips
 * (batched cost evaluations), batches.  Any output may be NULL. */
lsd_status_t lsd_galign_last_stats(lsd_galign_t* h, long long* launches, int* rounds, int* batches);
/* Lines :215-227 alone, pure host (works without a device): the output of lsd_sc_query for n_off offsets
 * (cand_idx / cand_dist / cand_shift [n_off][10], n_cand [n_off]) filtered by dist < dist_thres (detectCandidateMatch,
 * Scancontext.cpp:354) and merged per database index: the smaller float sc_dist wins, the first seen on a tie
 * (std::map<int, SCMatch>).  Out: ascending index, with float distance and yaw; *n_out = matches (may exceed cap). */
lsd_status_t lsd_galign_merge_candidates(const int32_t* cand_idx, const double* cand_dist, const int32_t* cand_shift,
                                         const int32_t* n_cand, int n_off, double dist_thres, int32_t* idx_out,
                                         float* dist_out, float* yaw_out, int cap, int* n_out);
/* Parity tap: FAST_VGICP of new_slot against each of ref_slots[n] from guesses16 (double [n,16]), then getFitnessScore.
 * serial = 0: batched as in lsd_galign_search; serial = 1: the same pairs one after another through the single-pair
 * kernels of lsd_reg on this handle's tables (the bit-exactness reference).  Per pair: final pose (double [n,16]),
 * converged, iterations, fitness.  Any output may be NULL.  *launches / *rounds: kernel launches and host round trips
 * (cost evaluations) of the matching. */
lsd_status_t lsd_galign_match(lsd_galign_t* h, int32_t new_slot, const int32_t* ref_slots, const double* guesses16, int n,
                              int serial, double* final16, int32_t* converged, int32_t* iterations, double* fitness,
                              long long* launches, int* rounds);
/* The LM iteration log of pair i of the last lsd_galign_match, same layout as lsd_reg_iteration_log. */
lsd_status_t lsd_galign_iteration_log(lsd_galign_t* h, int i, double* out4_per_iter, int cap_iters, int* n_iters);
/* One VGICP cost evaluation of new_slot against ref_slot at T16 through the batched kernel (parity tap, as lsd_reg_cost):
 * update != 0 = linearize (correspondences refreshed), else compute_error with the correspondences of the last update of
 * this pair.  H36 / b6 may be NULL. */
lsd_status_t lsd_galign_cost(lsd_galign_t* h, int32_t new_slot, int32_t ref_slot, const double* T16, int update, double* H36,
                             double* b6, double* err, int* n_corr);

/* ------------------------------------------------------------------------------------------
 * Overlap detector of map merging — replaces OverlapDetector::detect
 * (slam/localization/include/overlap_merge.hpp:38-304, called from MapLoader::mergeMapSLAM,
 * slam/localization/src/map_loader.cpp:118-137, when both maps share a GNSS origin).  Key-frame clouds (sensor frame) of
 * both maps are uploaded once into one device pool, addressed by slot, with their graph id (KeyFrame::mId).  A key
 * frame's NDT table, point map, filtered copy and that copy's point map are built on its first use as a target within a
 * call; lsd_overlap_detect releases them when it returns (their buffers are reused by the next call), so device memory
 * grows with the new key frames of one fragment, not with the size of the merge.
 * lsd_overlap_detect does, for all new key frames of a fragment: find_candidates on the host (:113-145), the inlier
 * prescreen of every (new, candidate) pair in one launch (:160-163), NDT_CUDA of every pair that passed with the
 * Levenberg-Marquardt loops of all pairs advanced together (one batched cost launch per round, each pair bit-identical
 * to lsd_reg's single-pair kernels on the same NDT table), getFitnessScore(25) of the converged pairs in one launch (:171), the best candidate
 * per new key frame (:172-183), then per new key frame with a best candidate the accumulated target, FAST_GICP and the
 * filtered fitness gate (:185-210).  graph_add_edge / graph_optimize / graph_sync_pose stay with the caller.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_overlap lsd_overlap_t;
typedef struct lsd_overlap_params {
  double distance_thresh;             /* 30.0 m between the key frames' translations (overlap_merge.hpp:46,132)          */
  int32_t candidate_link_dist;        /* 10: a candidate needs get_connection_count(..., 10) >= 10 (:47,133-134)        */
  int32_t max_candidate_num;          /* 3 candidates at most (:48,138)                                                 */
  double fitness_score_max_range;     /* 25.0, SQUARED distance as PCL compares it (:49,171,204)                        */
  double fitness_score_thresh;        /* 1.5: the finetune's filtered score must not exceed it (:50,205)                */
  double fitness_inlier_thresh;       /* 0.2: the prescreen's inlier ratio must reach it (:51,161)                      */
  double inlier_max_range;            /* 1.0, the prescreen's max_range (squared, :160)                                 */
  double filter_range;                /* 100.0: filter() keeps sqrtf(x*x + y*y) < this, in float (:226)                 */
  float filter_min_z;                 /* 0.5: and z > this (:227)                                                       */
  lsd_reg_params_t coarse;            /* lsd_reg_default_params(LSD_REG_NDT_P2D): "NDT_CUDA" (:54), no timeout          */
  lsd_reg_params_t accurate;          /* LSD_REG_GICP with max_corr_dist = 0.5, transformation_epsilon = 0.001 (:58-60)  */
} lsd_overlap_params_t;

typedef struct lsd_overlap_result {
  int32_t key1, key2;          /* Overlap(key1 = best candidate slot, key2 = new key frame slot) (:210)               */
  double relpose16[16];        /* registration_accurate->getFinalTransformation() (float) widened, row-major: new key
                                  frame -> best candidate                                                             */
  double score;                /* calc_fitness_score(accum, new, relpose, 25).first (:204)                             */
  double coarse_score;         /* the best candidate's NDT getFitnessScore(25) (:171)                                  */
} lsd_overlap_result_t;

/* What detect decided for each new key frame (no reference counterpart beyond its LOG_INFO lines). */
#define LSD_OVERLAP_NO_CANDIDATES 0   /* find_candidates returned nothing (:148-150)                                     */
#define LSD_OVERLAP_NO_MATCH 1        /* every candidate failed the prescreen or did not converge (:181-183)             */
#define LSD_OVERLAP_GICP_DIVERGED 2   /* the finetune did not converge (:200-202)                                        */
#define LSD_OVERLAP_GICP_REJECT 3     /* the finetune's filtered score is above fitness_score_thresh (:205-207)          */
#define LSD_OVERLAP_FOUND 4
typedef struct lsd_overlap_report {
  int32_t new_slot, decision;
  int32_t n_candidates, n_prescreened;   /* candidates found / those whose inlier ratio reached fitness_inlier_thresh   */
  int32_t best_slot;                     /* the coarse stage's choice, -1 = none                                         */
  int32_t n_accum;                       /* points of the accumulated finetune target (0 when there was no best)         */
  int32_t accum_incomplete;              /* the filtered accumulated target's point map refused points (searches scan it) */
  double best_score;                     /* its NDT score (DBL_MAX when none)                                            */
  double score;                          /* the finetune's filtered score (GICP_REJECT, FOUND), else 0                   */
} lsd_overlap_report_t;

void lsd_overlap_default_params(lsd_overlap_params_t* p);
lsd_status_t lsd_overlap_create(lsd_overlap_t** out, const lsd_overlap_params_t* p);
lsd_status_t lsd_overlap_destroy(lsd_overlap_t* h);
/* KeyFrame::mPoints ([n,4], sensor frame) uploaded once, with the key frame's graph id.  *slot = 0, 1, 2, ... in call order. */
lsd_status_t lsd_overlap_add_keyframe(lsd_overlap_t* h, const float* xyzi_host, int n, int32_t id, int32_t* slot);
/* OverlapDetector::detect(keyframes, new_keyframes) (:63-110).  poses16 = mOdom of EVERY slot ([n_slots,16], double,
 * row-major); keyframes = the loaded map's slots in mKeyFrames order (its first entry is what keyframe_id_map's default
 * 0 points at, :189); new_keyframes = the fragment's slots; edges = graph_get_edges as [n_e][2] (prev id, next id).
 * Writes up to cap overlaps in new key frame order; *n_found = overlaps found (may exceed cap). */
lsd_status_t lsd_overlap_detect(lsd_overlap_t* h, const double* poses16, const int32_t* keyframes, int n_kf,
                                const int32_t* new_keyframes, int n_new, const int32_t* edges, int n_e, lsd_overlap_result_t* out,
                                int cap, int* n_found);
/* Per new key frame of the last lsd_overlap_detect, in order.  out may be NULL. */
lsd_status_t lsd_overlap_last_reports(lsd_overlap_t* h, lsd_overlap_report_t* out, int cap, int* n);
/* Work of the last lsd_overlap_detect: kernel launches, and host round trips of the NDT stage (batched cost rounds).
 * *target_buffers: sets of target tables the handle owns (the most one call needed); *targets_held: those a slot holds
 * now (0 after lsd_overlap_detect).  Any output may be NULL. */
lsd_status_t lsd_overlap_last_stats(lsd_overlap_t* h, long long* launches, int* rounds, int* target_buffers, int* targets_held);
/* Hands back the tables the parity taps (lsd_overlap_fitness, lsd_overlap_match) built and kept; lsd_overlap_detect does
 * this itself when it returns. */
lsd_status_t lsd_overlap_release_targets(lsd_overlap_t* h);
/* find_candidates (:113-145), pure host (works without a device).  poses16 / ids = mOdom / mId of slots 0 .. n_slots - 1;
 * new_slot and every entry of keyframes must lie in that range (LSD_ERR_INVALID otherwise).  The 10-NN over the key
 * frames' translations uses float points and float squared distances ((dx dx + dy dy) + dz dz); equal distances keep the
 * order of `keyframes`.  get_connection_count is the reference's level-counted search (visited marked on pop).
 * *n_cand = candidates (slots, in 10-NN order; may exceed cap). */
lsd_status_t lsd_overlap_find_candidates(const lsd_overlap_params_t* p, const double* poses16, const int32_t* ids, int n_slots,
                                         const int32_t* keyframes, int n_kf, const int32_t* edges, int n_e, int32_t new_slot,
                                         int32_t* cand_out, int cap, int* n_cand);
/* (new->mOdom.inverse() * cand->mOdom).matrix().cast<float>() (:159): Isometry3d inverse and product in double, each
 * sum left to right, rounded to float.  Pure host. */
void lsd_overlap_guess(const double* T_new16, const double* T_cand16, float* guess16);
/* Eigen::Isometry3f(ndt_final).inverse().matrix() (:198), in float.  Pure host. */
void lsd_overlap_finetune_guess(const float* ndt_final16, float* guess16);
/* Parity tap: calc_fitness_score(target, source, T, max_range) (:225-263) through the batched kernel.  The target is
 * filtered in its own frame; the source is transformed by T in float (PCL's order, no fused multiply-add) and filtered;
 * each kept source point takes its exact nearest neighbour in the filtered target and counts when d2 <= max_range.
 * score = sum d2 / counted (DBL_MAX when none), inlier_ratio = counted / kept (0 when none).  *target_incomplete: the
 * filtered target's point map refused points, so every search scanned the whole filtered target.  Outputs may be NULL. */
lsd_status_t lsd_overlap_fitness(lsd_overlap_t* h, int32_t target_slot, int32_t source_slot, const float* T16, double max_range,
                                 double* score, double* inlier_ratio, int* n_counted, int* n_filtered, int* target_incomplete);
/* Parity tap: the coarse stage alone for an explicit pair list (new_slots[i] is the NDT target, cand_slots[i] the source,
 * guesses16 double [n,16]); the pairs may span several targets.  serial = 0: batched as in lsd_overlap_detect; serial = 1:
 * the same pairs one after another through the single-pair kernels of lsd_reg on this handle's tables (the bit-exactness
 * reference: a separate lsd_reg handle builds its own NDT table, whose double atomic sums may differ in the last bits
 * from build to build).  Per pair: final NDT pose (double [n,16]),
 * converged, iterations, getFitnessScore(fitness_score_max_range) at that pose (DBL_MAX when not converged).  Any output
 * may be NULL.  *launches / *rounds: kernel launches and host round trips (batched cost evaluations) of the call. */
lsd_status_t lsd_overlap_match(lsd_overlap_t* h, const int32_t* new_slots, const int32_t* cand_slots, const double* guesses16, int n,
                               int serial, double* final16, int32_t* converged, int32_t* iterations, double* fitness, long long* launches, int* rounds);
/* The LM iteration log of pair i of the last lsd_overlap_match / detect, same layout as lsd_reg_iteration_log. */
lsd_status_t lsd_overlap_iteration_log(lsd_overlap_t* h, int i, double* out4_per_iter, int cap_iters, int* n_iters);

/* ------------------------------------------------------------------------------------------
 * Detection voxelizer (config 5) — replaces sensor_driver/inference/voxelize:
 * Preprocess::forward (preprocess_kernel.cu:56-101: sliding window of max_frame_num frames, older frames
 * re-projected by a 3x4 motion, time channel + 0.1) and Voxelization::forward (voxelization_kernel.cu:
 * 225-255: hash voxelisation, <= max_points_per_voxel points per voxel, mean -> fp16).  Output rows are in
 * order of each voxel's first point; features [V, num_feature] fp16, indices [V,4] u32 = (0, z, y, x) or
 * (0, x, y, z).  The closed libspconv engine that consumes them is out of scope (SURVEY F5).
 * The window keeps the reference's counts: a realtime frame gets at least one row even when the other frames fill
 * max_points, so the total (and lsd_vfe_get_points) can reach max_points + max_frame_num - 1 rows.  A NaN coordinate
 * passes the range test and lands in cell 0 of its axis, as in the reference.  Deviations from the reference:
 *   - an empty realtime frame (num_points = 0, points_host may be NULL) reads nothing from the caller; the one row the
 *     reference counts for it (and copies from the caller's array) is written as (1e30, 1e30, 1e30, 0, ...), which no
 *     rigid motion brings into a range box;
 *   - the window transform carries every feature past z and adds 0.1 to feature 4 only when num_feature > 4 (the
 *     reference copies features 3 and 4 whatever num_feature is);
 *   - a cell that only the range test rejects (a max face inside a grid rounded up) yields no row; the reference emits a
 *     row of NaN features for it;
 *   - realtime = 0 empties every frame slot (the reference's resize keeps the older slots' counts, so its next realtime
 *     frame subtracts rows that are no longer in the window);
 *   - lsd_vfe_create returns LSD_ERR_INVALID for a grid of 2^31 cells or more (voxel keys are 32-bit).
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_vfe lsd_vfe_t;
typedef struct lsd_vfe_params {
  float min_range[3], max_range[3], voxel_size[3];  /* [-64,-64,-2 .. 64,64,4], 0.1 x 0.1 x 0.15 (detection_object.yaml:7-16) */
  int max_points_per_voxel;                          /* 5   (inference.h:16-38) */
  int max_voxels;                                    /* 300000 */
  int max_points;                                    /* 500000 */
  int num_feature;                                   /* 5: x, y, z, intensity, time */
  int max_frame_num;                                 /* POINT_FRAME_NUM 2 (README's best model: 4) */
  int unordered_ids;        /* 0 (default): voxel ids in the order of each voxel's first point (deterministic: one extra scan
                               kernel); 1: ids in atomic order like the reference's voxelization_kernel (same voxel SET and rows,
                               any numbering): two kernels instead of three */
} lsd_vfe_params_t;
void lsd_vfe_default_params(lsd_vfe_params_t* p);
lsd_status_t lsd_vfe_create(lsd_vfe_t** out, const lsd_vfe_params_t* p);
lsd_status_t lsd_vfe_destroy(lsd_vfe_t* v);
lsd_status_t lsd_vfe_accumulate(lsd_vfe_t* v, const float* points_host, int num_points, const float* motion16_host, int realtime,
                                int* total_points);
lsd_status_t lsd_vfe_voxelize(lsd_vfe_t* v, int order_zyx, int* num_voxels);
lsd_status_t lsd_vfe_get_output(lsd_vfe_t* v, void* features_fp16_host, unsigned* indices_host, unsigned* num_points_host);
lsd_status_t lsd_vfe_get_output_dev(lsd_vfe_t* v, const void** features_fp16, const unsigned** indices, const unsigned** num_points);
lsd_status_t lsd_vfe_get_points(lsd_vfe_t* v, float* points_host, int cap, int* total);

/* ------------------------------------------------------------------------------------------
 * IMU forward propagation + per-point undistortion — replaces ImuProcess
 * (slam/mapping/fastlio/src/IMU_Processing.hpp:28-450; called at laserMapping.cpp:1188) and
 * esekf::predict (IKFoM_toolkit/esekfom/esekfom.hpp:279-383 with use-ikfom.hpp:36-88).
 *   imu7: double [n_imu, 7] = (stamp s, gyr xyz rad/s, acc xyz in units of g) — MeasureGroup::imu;
 *   ins_vel3: MeasureGroup::ins.back() (Ve, Vn, Vu) or NULL; lidar_beg/end_time: MeasureGroup's;
 *   xyzi [n,4] + time_ms [n] (PointType::curvature, ms since lidar_beg_time): MeasureGroup::lidar.
 * lsd_imu_process = ImuProcess::Process: LSD_IMU_INITIALIZING while the first MAX_INI_COUNT (100) IMU
 * samples are being averaged (state/P are initialised as IMU_init does), then LSD_OK with the state and
 * covariance propagated to the scan end and the undistorted cloud left on the device
 * (lsd_imu_get_cloud_dev) ready for lsd_lio_scan_dev.  Points stay in INPUT order (the reference sorts by
 * time; nothing downstream depends on the order).  Forward propagation runs on the host in double like the
 * reference; the backward propagation of the points is one kernel.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_imu lsd_imu_t;
typedef struct lsd_imu_params {
  double ext_R[9], ext_t[3];                     /* Lidar_R_wrt_IMU (row-major), Lidar_T_wrt_IMU: set_extrinsic          */
  double gyr_cov, acc_cov, b_gyr_cov, b_acc_cov; /* 0.1, 0.1, 1e-4, 1e-4 (laserMapping.cpp:1076-1079, :1102-1105)       */
  int undistort;                                 /* fastlio_init(..., undistort), laserMapping.cpp:1106                  */
} lsd_imu_params_t;
void lsd_imu_default_params(lsd_imu_params_t* p);
lsd_status_t lsd_imu_create(lsd_imu_t** out, const lsd_imu_params_t* p);
lsd_status_t lsd_imu_destroy(lsd_imu_t* m);
lsd_status_t lsd_imu_reset(lsd_imu_t* m);                         /* ImuProcess::Reset + first-frame flag */
lsd_status_t lsd_imu_is_init(lsd_imu_t* m, int* flag);            /* ImuProcess::IsInit */
lsd_status_t lsd_imu_process(lsd_imu_t* m, const double* imu7, int n_imu, const double* ins_vel3_or_null, double lidar_beg_time,
                             double lidar_end_time, const float* xyzi_host, const float* time_ms_host, int n, double* state26_inout,
                             double* P529_inout, int* n_out);
lsd_status_t lsd_imu_process_dev(lsd_imu_t* m, const double* imu7, int n_imu, const double* ins_vel3_or_null, double lidar_beg_time,
                                 double lidar_end_time, const float* xyzi_dev, const float* time_ms_dev, int n, double* state26_inout,
                                 double* P529_inout, int* n_out);
/* The undistorted cloud of the last lsd_imu_process call; *cuda_stream_out (may be NULL) is the stream it
 * is produced on — synchronise it (or use lsd_imu_get_cloud) before reading from another stream. */
lsd_status_t lsd_imu_get_cloud_dev(lsd_imu_t* m, const float** xyzi_dev, int* n, void** cuda_stream_out);
lsd_status_t lsd_imu_get_cloud(lsd_imu_t* m, float* xyzi_host, int cap, int* n);
/* Parity tap: the IMUpose list of the last scan, double [n, 22] = (offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]). */
lsd_status_t lsd_imu_get_poses(lsd_imu_t* m, double* poses22, int cap, int* n);
/* ImuProcess::start_state_point (the state at the scan start, IMU_Processing.hpp:234,266) and mean_acc_norm (:206): what
 * fastlio_state() and fastlio_odometry() hand to the caller (laserMapping.cpp:690-738).  Host only. */
lsd_status_t lsd_imu_get_start_state(lsd_imu_t* m, double* state26, double* mean_acc_norm);
/* esekf::predict alone (host, no GPU): Q144 = 12x12 process noise (ng, na, nbg, nba). */
lsd_status_t lsd_eskf_predict(double* state26_inout, double* P529_inout, double dt, const double* Q144, const double* acc3,
                              const double* gyro3);

/* ------------------------------------------------------------------------------------------
 * Key-frame cloud filters (row N3) — replaces, for every new key frame (slam/src/slam.cpp:398-410):
 * pcl::RadiusOutlierRemoval with setRadiusSearch(radius = 1.0) / setMinNeighborsInRadius(min_neighbors = 3)
 * (slam.cpp:104-108: a point stays iff its radius search, which includes the point itself, returns MORE than
 * min_neighbors points) followed by pointsDistanceFilter(cloud, out, min_range = 0, max_range = key_frame_range)
 * (slam_utils.cpp:236-247: min < |x| < max and min < |y| < max).  Order preserving.  radius == 0 skips the
 * outlier test.  out must hold n points; *n_out = points kept.
 * ------------------------------------------------------------------------------------------ */
lsd_status_t lsd_keyframe_filter(const float* xyzi_host, int n, float radius, int min_neighbors, float min_range, float max_range,
                                 float* out_host, int* n_out);
lsd_status_t lsd_keyframe_filter_dev(const float* xyzi_dev, int n, float radius, int min_neighbors, float min_range, float max_range,
                                     float* out_dev, int* n_out);

/* ------------------------------------------------------------------------------------------
 * Key-frame files (row N3) — the on-disk format the reference's map editor and map loader read.
 * lsd_keyframe_save == dump_keyframe (slam/src/graph_utils.cpp:123-131, bound at slam/src/slam_wrapper.cpp:273) ->
 * KeyFrame::save (slam/common/keyframe.cpp:118-132): <directory>/cloud.pcd, a PCL binary PCD of PointXYZI (fields
 * x y z intensity, 16 bytes per point; an empty cloud gets the ASCII header of slam/common/pcd_writer.cpp:9-25), with the
 * intensity multiplied by 255 (numpy_to_pointcloud(points, 255.0)), and <directory>/data:
 *     stamp <sec> <nsec>\n estimate\n <4x4>\n odom \n <4x4>\n id <id>\n
 * the matrices exactly as Eigen prints them (6 significant digits, columns right-aligned to a common width).
 * lsd_keyframe_load == KeyFrame(id, directory, true) + loadOdom + loadPcd (keyframe.cpp:18-106): timestamp in us, the
 * "estimate" matrix, intensity / 255.  pose16: row-major 4x4 doubles.  The directory must exist (the caller makes it,
 * slam/map_manager.py:286-288).  Host-only: no device is touched.
 * ------------------------------------------------------------------------------------------ */
lsd_status_t lsd_keyframe_save(const char* directory, uint64_t stamp_us, int64_t id, const float* xyzi_host, int n,
                               const double* pose16);
/* xyzi_out may be NULL to query *n; cap = points xyzi_out can hold (LSD_ERR_CAPACITY if the file has more). */
lsd_status_t lsd_keyframe_load(const char* directory, uint64_t* stamp_us, int64_t* id, double* pose16, float* xyzi_out, int cap,
                               int* n);

/* ------------------------------------------------------------------------------------------
 * Local-map assembly for localisation (row N2) — replaces the body of Localization::runUpdateLocalMap
 * (slam/localization/src/localization.cpp:303-373): key frames within 30 m of the pose, nearest first, thinned by
 * key_frame_distance, concatenated up to 200 000 points, VoxelGrid at max(resolution, 0.1).  Key-frame clouds are
 * uploaded once (lsd_localmap_add_keyframe: mTransfromPoints, map frame) and stay on the device; the assembled map
 * is handed to the matcher without leaving it: lsd_localmap_get_dev -> lsd_reg_set_target_dev (updateLocalMap).
 * lsd_localmap_update returns LSD_LOCALMAP_NONE where the reference sets mLocalMap = nullptr (no key frame in
 * range, or the nearest one >= 20 m away).  The 10 m update hysteresis stays with the caller (:325-327).
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_localmap lsd_localmap_t;
lsd_status_t lsd_localmap_create(lsd_localmap_t** out, double resolution, double key_frame_distance);
lsd_status_t lsd_localmap_destroy(lsd_localmap_t* h);
lsd_status_t lsd_localmap_add_keyframe(lsd_localmap_t* h, const float* xyzi_map_host, int n, const double* position3);
lsd_status_t lsd_localmap_update(lsd_localmap_t* h, const double* pose_xyz, int* n_points, int* n_keyframes_in_radius, double* nearest_dist);
lsd_status_t lsd_localmap_get_dev(lsd_localmap_t* h, const float** xyzi_dev, int* n);
lsd_status_t lsd_localmap_get(lsd_localmap_t* h, float* xyzi_host, int cap, int* n);

/* ------------------------------------------------------------------------------------------
 * The LIO seam (SURVEY.md 8b "C++ seam 1") — the eight free functions slam/mapping/fastlio/src/fastlio.cpp:9-16 binds,
 * with the reference's file-scope state (laserMapping.cpp:60-200) in a handle.  Same contract: any thread may enqueue,
 * one consumer thread calls lsd_fastlio_main (fastlio.cpp:263-277).
 *   fastlio_init(extT, extR, filter_num, max_point_num, scan_period, undistort)   -> lsd_fastlio_create   (:1025-1124)
 *   fastlio_imu_enqueue(ImuType)              -> lsd_fastlio_imu_enqueue (stamp s, gyr rad/s, acc m/s^2; / 9.81 inside, :414)
 *   fastlio_ins_enqueue(bool, RTKType)        -> lsd_fastlio_ins_enqueue (ENU velocity, heading / pitch / roll in degrees, :418-443)
 *   fastlio_pcl_enqueue(PointCloudAttrPtr&)   -> lsd_fastlio_pcl_enqueue (xyzi [n,4], PointAttr::stamp [n] in us relative to the
 *                                                header stamp; Preprocess::velodyne_handler's decimation and blind zone inside)
 *   fastlio_main()                            -> lsd_fastlio_main: 1 = a package was consumed, 0 = nothing ready, < 0 = error
 *   fastlio_odometry(odom_s, odom_e)          -> lsd_fastlio_odometry (row-major 4x4)
 *   fastlio_state()                           -> lsd_fastlio_state (20 doubles, :714-738)
 *   fastlio_is_init()                         -> lsd_fastlio_is_init
 * lsd_fastlio_main = sync_packages (:445-520) -> ImuProcess::Process (lsd_imu_process) -> flg_EKF_inited, NEARBY74 -> NEARBY18
 * after 1 s -> lsd_lio_scan_dev with the reference's stale Nearest_Points rows on.  The engines are created on the first
 * package that needs them; everything before that (queues, decimation, package synchronisation) is host code and works
 * without a device — lsd_fastlio_pop_package is the parity tap on it.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_fastlio lsd_fastlio_t;
lsd_status_t lsd_fastlio_create(lsd_fastlio_t** out, const double* extT3, const double* extR9, int filter_num, int max_point_num,
                                double scan_period, int undistort);
/* optional, before the first lsd_fastlio_main: map table size (default 2^22 lines) and raw scan capacity (default 262144) */
lsd_status_t lsd_fastlio_set_capacity(lsd_fastlio_t* f, int map_log2_lines, int max_scan_points);
lsd_status_t lsd_fastlio_destroy(lsd_fastlio_t* f);
lsd_status_t lsd_fastlio_imu_enqueue(lsd_fastlio_t* f, double stamp_s, const double* gyr3, const double* acc3);
lsd_status_t lsd_fastlio_ins_enqueue(lsd_fastlio_t* f, int rtk_valid, int is_wheel, uint64_t timestamp_us, const double* vel_enu3,
                                     double heading_deg, double pitch_deg, double roll_deg);
lsd_status_t lsd_fastlio_pcl_enqueue(lsd_fastlio_t* f, const float* xyzi, const uint32_t* stamp_us, int n, uint64_t header_stamp_us);
int lsd_fastlio_main(lsd_fastlio_t* f);
lsd_status_t lsd_fastlio_odometry(lsd_fastlio_t* f, double* odom_start16, double* odom_end16);
lsd_status_t lsd_fastlio_state(lsd_fastlio_t* f, double* out20);
int lsd_fastlio_is_init(lsd_fastlio_t* f);
/* What the last lsd_fastlio_main did: the lsd_lio_scan status (LSD_OK, LSD_MAP_SEEDED, LSD_SCAN_TOO_SMALL,
 * LSD_NO_EFFECTIVE_POINTS) or LSD_IMU_INITIALIZING, and the scan's counters; kf.get_x() / kf.get_P(); the LIO handle. */
lsd_status_t lsd_fastlio_last(lsd_fastlio_t* f, int* status, lsd_lio_info_t* info);
lsd_status_t lsd_fastlio_get_filter(lsd_fastlio_t* f, double* state26, double* P529);
lsd_lio_t* lsd_fastlio_lio(lsd_fastlio_t* f);
/* Parity tap, host only: sync_packages alone — pops the next package instead of processing it.  1 = filled, 0 = none ready. */
int lsd_fastlio_pop_package(lsd_fastlio_t* f, double* lidar_beg_time, double* lidar_end_time, int* n_points, float* xyzi, float* time_ms,
                            int cap_points, int* n_imu, double* imu7, int cap_imu, int* have_ins, double* ins_vel3);

/* ------------------------------------------------------------------------------------------
 * ScanContext (row N4) — replaces SCManager (slam/common/Scancontext/Scancontext.h:44-98, Scancontext.cpp) as used by
 * KeyFrame::computeDescriptor (slam/common/keyframe.cpp:165-167), GlobalLocalization::setInitPoseRange / localSearch /
 * globalSearch / imageSearch (slam/localization/src/global_localization.cpp:104-118,350-398,439-441) and global_alignment
 * (slam/localization/include/global_alignment.hpp:206-237).  A descriptor is 20 rings x 60 sectors of doubles in Eigen's
 * own storage order (column-major, MatrixXd::data(): element (ring, sector) at sector * 20 + ring); ring keys are the
 * row means (20), sector keys the column means (60).  The database (buildRingKeyKDTree's polarcontexts_ + ring-key tree)
 * lives on the device.  Descriptors are bit-exact; keys and distances follow Eigen's reduction order.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_sc lsd_sc_t;
#define LSD_SC_MAX_QUERIES 64 /* descriptors made / queried per call */
#define LSD_SC_CANDIDATES 10  /* NUM_CANDIDATES_FROM_TREE, Scancontext.h:78 */
lsd_status_t lsd_sc_create(lsd_sc_t** out, int db_capacity);
lsd_status_t lsd_sc_destroy(lsd_sc_t* s);
/* SCManager::makeScancontext(cloud, dx, dy) + makeRingkey / makeSectorkeyFromScancontext for n_off offsets of ONE cloud
 * in one pass (offsets_xy [n_off][2]; NULL = the single offset (0, 0); the reference's search_trans has 9).  Outputs may
 * be NULL: desc_out [n_off][1200], ringkey_out [n_off][20], sectorkey_out [n_off][60].  The descriptors stay on the
 * device as query slots 0..n_off-1 for lsd_sc_query(NULL), lsd_sc_detect_* and lsd_sc_db_add_made. */
lsd_status_t lsd_sc_make(lsd_sc_t* s, const float* xyzi_host, int n, const double* offsets_xy, int n_off, double* desc_out,
                         double* ringkey_out, double* sectorkey_out);
lsd_status_t lsd_sc_make_dev(lsd_sc_t* s, const float* xyzi_dev, int n, const double* offsets_xy, int n_off, double* desc_out,
                             double* ringkey_out, double* sectorkey_out);
/* buildRingKeyKDTree(polarcontext_invkeys_mat, polarcontexts): clear, then add the key frames' descriptors (their ring
 * keys are recomputed on the device); lsd_sc_db_add_made appends query slot `slot` of the last lsd_sc_make without a
 * host round trip.  Database index = order of insertion. */
lsd_status_t lsd_sc_db_clear(lsd_sc_t* s);
lsd_status_t lsd_sc_db_add(lsd_sc_t* s, const double* desc_host, int n);
lsd_status_t lsd_sc_db_add_made(lsd_sc_t* s, int slot);
lsd_status_t lsd_sc_db_size(lsd_sc_t* s, int* n);
/* The retrieval common to detectClosestMatch and detectCandidateMatch (Scancontext.cpp:280-299): for each of nq queries
 * (desc_host [nq][1200], or NULL = the slots of the last lsd_sc_make) the min(10, database size) entries with the
 * nearest ring keys, ascending, each scored with distanceBtnScanContext.  cand_idx / cand_dist / cand_shift are
 * [nq][10], padded with -1 / 1e7 / 0; n_cand [nq]. */
lsd_status_t lsd_sc_query(lsd_sc_t* s, const double* desc_host_or_null, int nq, int32_t* cand_idx, double* cand_dist, int32_t* cand_shift,
                          int32_t* n_cand);
/* SCManager::distanceBtnScanContext(sc1, sc2) for n_pairs pairs (localSearch, imageSearch): dist, argmin shift. */
lsd_status_t lsd_sc_distance(lsd_sc_t* s, const double* desc_a_host, const double* desc_b_host, int n_pairs, double* dist, int32_t* shift);
/* detectClosestMatch / detectCandidateMatch for query slot `slot`: loop id (-1: none below dist_thres = SC_DIST_THRES),
 * yaw = deg2rad(shift * 6 deg), score = the smallest distance (untouched on an empty database, like the reference). */
lsd_status_t lsd_sc_detect_closest(lsd_sc_t* s, int slot, double dist_thres, int32_t* loop_id, float* yaw_rad, double* score);
lsd_status_t lsd_sc_detect_candidates(lsd_sc_t* s, int slot, double dist_thres, int32_t* idx10, float* yaw10, float* dist10, int32_t* n);

/* ------------------------------------------------------------------------------------------
 * Floor detection — replaces FloorDetectionNodelet::detect (slam/backend/hdl_graph_slam/apps/floor_detection_nodelet.cpp:79-193)
 * after PrefilteringNodelet (prefiltering_nodelet.cpp:91-165), the per-frame work of FastLIO's "FLIO Floor" thread
 * (slam/mapping/fastlio/src/fastlio.cpp:279-292), and the two detect_ground copies (slam/src/graph_utils.cpp:329-382,
 * slam/localization/map_render/map_render.cpp:81-134).  One call = one frame on the handle's own stream: VoxelGrid + distance
 * filter (optional), the two PlaneClipper3D height clips, NormalEstimation (k = 10) + the |n_z| filter, and
 * RandomSampleConsensus with SampleConsensusModelPlane (PCL 1.9.1, boost::mt19937 seeded 12345 on every call, so the floor
 * is a pure function of the cloud).  The rules are restated in DESIGN.md section 5f.  A handle is confined to one host
 * thread at a time; handles on different threads (and an lsd_lio_t / lsd_fastlio_t) run side by side.
 * ------------------------------------------------------------------------------------------ */
typedef struct lsd_floor lsd_floor_t;
#define LSD_FLOOR_MAPPING 0   /* prefiltering_nodelet + FloorDetectionNodelet: leaf 0.2, 0.1 < d < 100, clip 2.0 / -1.0      */
#define LSD_FLOOR_GROUND 1    /* graph_utils.cpp::detect_ground: no prefilter, clip 1.5 / -1.5, threshold 0.1, inlier cloud    */
#define LSD_FLOOR_RENDER 2    /* map_render.cpp::detect_ground: as GROUND with a RANSAC threshold of 0.2                      */
typedef struct lsd_floor_params {
  float prefilter_leaf;             /* VoxelGrid leaf of the prefilter (0 = no prefilter, and no distance filter)             */
  double distance_near, distance_far; /* distance filter d > near && d < far, d = double(float |xyz|) (:152-155)             */
  float clip_keep_d;                /* keep z >= -clip_keep_d (plane (0, 0, 1, d), ExtractIndices negative = false)          */
  float clip_cut_d;                 /* then drop z >= -clip_cut_d (ExtractIndices negative = true)                           */
  int use_normal_filtering;         /* 1 (floor_detection_nodelet.cpp:44)                                                   */
  int normal_k;                     /* 10 (setKSearch(10)); no other value is supported                                     */
  double normal_filter_deg;         /* keep |n_z| > cos(20 deg)                                                             */
  float viewpoint_z;                /* setViewPoint(0, 0, sensor_height = 0): the sign of the normals only                  */
  double ransac_threshold;          /* setDistanceThreshold: 0.1 (0.2 for RENDER)                                           */
  double ransac_probability;        /* 0.99, SampleConsensus default                                                        */
  int ransac_max_iterations;        /* 10000, SampleConsensus default                                                       */
  int floor_pts_thresh;             /* 1024: fewer candidates or inliers = no floor                                         */
  double floor_normal_deg;          /* 10: |c2| < cos(10 deg) = not vertical                                                */
  int hypotheses_per_batch;         /* hypotheses drawn and scored per launch pair (256, 1 .. 12288); no output depends on it */
} lsd_floor_params_t;

#define LSD_FLOOR_FOUND 0
#define LSD_FLOOR_EMPTY 1             /* the input cloud is empty                                                            */
#define LSD_FLOOR_FEW_CANDIDATES 2    /* fewer than floor_pts_thresh points after the clip and the normal filter (:91-93)    */
#define LSD_FLOOR_NO_MODEL 3          /* RANSAC found no model (no sample could be drawn, or fewer than 3 candidates)       */
#define LSD_FLOOR_FEW_INLIERS 4       /* fewer than floor_pts_thresh inliers (:105-107)                                      */
#define LSD_FLOOR_NOT_VERTICAL 5      /* |c2| < cos(floor_normal_deg) (:115-119)                                             */
typedef struct lsd_floor_result {
  int32_t found, reason;            /* reason: LSD_FLOOR_*                                                                   */
  float coeffs[4];                  /* the plane, c2 >= 0 when found (:122-124); RANSAC's best model otherwise              */
  int32_t n_input, n_prefiltered, n_clipped, n_candidates, n_inliers;
  int32_t map_dropped;              /* points the normals' point map refused: every point then took the exact scan        */
  int32_t iterations, skipped;      /* RandomSampleConsensus's iterations_ and skipped_count at the stop                   */
  int32_t best_hypothesis;          /* draw-order index of the best model (-1: none)                                       */
  int32_t batches;                  /* sampler + scoring launch pairs                                                      */
  int64_t hypotheses_scored;        /* batches x hypotheses_per_batch                                                      */
  int32_t launches, round_trips;    /* kernel launches and host waits of the call                                         */
} lsd_floor_result_t;

#define LSD_FLOOR_STAGE_PREFILTERED 0
#define LSD_FLOOR_STAGE_CLIPPED 1
#define LSD_FLOOR_STAGE_CANDIDATES 2
#define LSD_FLOOR_STAGE_INLIERS 3

void lsd_floor_default_params(lsd_floor_params_t* p, int preset);
lsd_status_t lsd_floor_create(lsd_floor_t** out, const lsd_floor_params_t* p);
lsd_status_t lsd_floor_destroy(lsd_floor_t* f);
/* One frame ([n,4] xyzi, sensor frame).  The device entry reads xyzi_dev on the handle's stream. */
lsd_status_t lsd_floor_detect(lsd_floor_t* f, const float* xyzi_host, int n, lsd_floor_result_t* res);
lsd_status_t lsd_floor_detect_dev(lsd_floor_t* f, const float* xyzi_dev, int n, lsd_floor_result_t* res);
/* The cloud of a stage of the last call (LSD_FLOOR_STAGE_*), in order; INLIERS is detect_ground's output cloud.
 * Writes up to cap points; *n = the stage's size.  The _dev form returns a device pointer valid until the next detect. */
lsd_status_t lsd_floor_get_cloud(lsd_floor_t* f, int stage, float* out, int cap, int* n);
lsd_status_t lsd_floor_get_cloud_dev(lsd_floor_t* f, int stage, const float** xyzi_dev, int* n);
/* Per clipped point of the last call: the normal and curvature (nx, ny, nz, curvature) after flipNormalTowardsViewpoint,
 * and the fp32 covariance (xx, xy, xz, yy, yz, zz) of its 10 neighbours.  NaN for fewer than 3 neighbours.  Either output
 * may be NULL; *n = clipped points (0 without normal filtering). */
lsd_status_t lsd_floor_get_normals(lsd_floor_t* f, float* normal4, float* cov6, int cap, int* n);
/* The hypotheses RANSAC drew in the last call, in draw order, up to the stop: candidate indices [n,3], flag (1 model,
 * 0 collinear = skipped, -1 no sample could be drawn) and inlier count.  Any output may be NULL. */
lsd_status_t lsd_floor_last_samples(lsd_floor_t* f, int32_t* idx3, int32_t* flags, int32_t* counts, int cap, int* n);
/* The stop rule of RandomSampleConsensus::computeModel, pure host (works without a device), on hypotheses in draw order
 * (inlier counts and flags as lsd_floor_last_samples gives them) over a cloud of n_points: *consumed = hypotheses drawn
 * before the loop ended (-1: it had not ended after n), *best = index of the best model (-1: none), *iterations /
 * *skipped = iterations_ / skipped_count (either may be NULL). */
lsd_status_t lsd_ransac_replay(const int32_t* counts, const int32_t* flags, int n, int n_points, double probability,
                               int max_iterations, int* consumed, int* best, int* iterations, int* skipped);

/* Host-side manifold helpers (exported so bindings/tests use the same algebra as the filter).
 * IMU_Processing.hpp:224-230 initial covariance; state_ikfom boxplus/boxminus. */
void lsd_lio_init_cov(double* P529);
void lsd_state_boxplus(double* state26_inout, const double* delta23);
void lsd_state_boxminus(const double* a26, const double* b26, double* out23);
/* The filter alone, on the host (no GPU): runs esekf::update_iterated_dyn_share_modified with the
 * measurement model replaced by a caller-supplied table — evaluation e uses HTH36[e], HTh6[e],
 * n_eff[e] (n_eff[e] < 1 = invalid).  Returns the number of evaluations consumed; converge_log16_or_null[e] receives
 * the `converge` flag evaluation e was called with (what h_share_model reads to decide on a new neighbour search,
 * laserMapping.cpp:838-852).  Used by the CPU
 * test-suite to check the host algebra against the oracle without a device. */
int lsd_eskf_update_table(double* state26_inout, double* P529_inout, const double* HTH36, const double* HTh6,
                          const int* n_eff, int n_table, double R, int max_iterations, double eps, int literal,
                          int* converge_log16_or_null);

#ifdef __cplusplus
}
#endif
#endif /* LSDREG_H */
