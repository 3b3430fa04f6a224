"""TEST INFRASTRUCTURE ONLY — ctypes bindings for the CPU oracle.

Two libraries (built by oracle/Makefile):
  liblsd_oracle.so      our plain-C restatement ("port") of the reference algorithms
  _ref/libref_lio.so    the UNMODIFIED reference sources (iVox, ikd-Tree, esti_plane) compiled
                        where they lie under /root/reference ("reference")

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT = os.path.join(_HERE, "liblsd_oracle.so")
_REF = os.path.join(_HERE, "_ref", "libref_lio.so")

_f = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_d = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_i = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_u8 = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


def _load_port():
    if not os.path.exists(_PORT):
        raise RuntimeError(f"{_PORT} missing: run `make -C oracle` (or __graft_entry__.build())")
    L = C.CDLL(_PORT)
    L.orc_voxelgrid.restype = C.c_int
    L.orc_voxelgrid.argtypes = [_f, C.c_int, C.c_float, _f, C.c_void_p]
    L.orc_ivox_create.restype = C.c_void_p
    L.orc_ivox_create.argtypes = [C.c_float, C.c_int, C.c_size_t]
    L.orc_ivox_set_nearby.argtypes = [C.c_void_p, C.c_int]
    L.orc_ivox_destroy.argtypes = [C.c_void_p]
    L.orc_ivox_num_cells.restype = C.c_size_t
    L.orc_ivox_num_cells.argtypes = [C.c_void_p]
    L.orc_ivox_num_points.restype = C.c_size_t
    L.orc_ivox_num_points.argtypes = [C.c_void_p]
    L.orc_ivox_add.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.orc_ivox_delete_boxes.restype = C.c_size_t
    L.orc_ivox_delete_boxes.argtypes = [C.c_void_p, _f, C.c_int]
    L.orc_knn.argtypes = [C.c_void_p, C.c_int, _f, C.c_int, C.c_int, C.c_int, C.c_double, _i, _f, _f, _i, C.c_int]
    L.orc_esti_plane_batch.argtypes = [_f, C.c_int, C.c_float, _f, _i]
    L.orc_lio_hmodel.restype = C.c_int
    L.orc_lio_hmodel.argtypes = [C.c_void_p, _f, C.c_int, _d, _d, _d, _d, C.c_int, C.c_int, _f, _i, _i, _u8,
                                 _f, _f, _d, _d, _d, _i, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L.orc_ndt_build.restype = C.c_void_p
    L.orc_ndt_build.argtypes = [_f, C.c_int, C.c_int, C.c_float]
    L.orc_ndt_destroy.argtypes = [C.c_void_p]
    L.orc_ndt_num_voxels.restype = C.c_size_t
    L.orc_ndt_num_voxels.argtypes = [C.c_void_p]
    L.orc_ndt_voxel.restype = C.c_int
    L.orc_ndt_voxel.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _f, _f]
    L.orc_ndt_cost.restype = C.c_double
    L.orc_ndt_cost.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, _d, _d, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_gicp_normals.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, C.c_int, C.c_double, _d, _i, C.c_int]
    L.orc_gicp_cost.restype = C.c_double
    L.orc_gicp_cost.argtypes = [C.c_void_p, _f, C.c_int, _d, _f, C.c_int, _d, C.c_int, _d, C.c_double, C.c_int, _i, _d,
                                C.c_void_p, C.c_void_p, C.c_int]
    L.orc_vgicp_build.restype = C.c_void_p
    L.orc_vgicp_build.argtypes = [_f, C.c_int, C.c_int, _d, C.c_double]
    L.orc_vgicp_destroy.argtypes = [C.c_void_p]
    L.orc_vgicp_num_voxels.restype = C.c_size_t
    L.orc_vgicp_num_voxels.argtypes = [C.c_void_p]
    L.orc_vgicp_voxel.restype = C.c_int
    L.orc_vgicp_voxel.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _d, _d]
    L.orc_vgicp_cost.restype = C.c_double
    L.orc_vgicp_cost.argtypes = [C.c_void_p, _f, C.c_int, _d, C.c_int, _d, C.c_int, C.c_int,
                                 np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS"), _d, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_fitness.restype = C.c_double
    L.orc_fitness.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, _d, C.c_double, C.c_double]
    L.orc_map_incremental.restype = C.c_int
    L.orc_map_incremental.argtypes = [C.c_void_p, _f, C.c_int, _d, _d, _d, _d, _f, _i, C.c_int, C.c_double, _f, _u8, C.c_int, C.c_int]
    return L


def _load_ref():
    if not os.path.exists(_REF):
        return None
    L = C.CDLL(_REF)
    L.ref_ivox_create.restype = C.c_void_p
    L.ref_ivox_create.argtypes = [C.c_float, C.c_int, C.c_size_t, C.c_double]
    L.ref_ivox_destroy.argtypes = [C.c_void_p]
    L.ref_ivox_add.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, C.c_double]
    L.ref_ivox_num_cells.restype = C.c_size_t
    L.ref_ivox_num_cells.argtypes = [C.c_void_p]
    if hasattr(L, "ref_ivox_dump"):        # a library built from an older ref_lio.cpp lacks them (see HAVE_REF_IVOX_DUMP)
        L.ref_ivox_add_ids.argtypes = [C.c_void_p, _f, _i, C.c_int, C.c_double]
        L.ref_ivox_num_points.restype = C.c_size_t
        L.ref_ivox_num_points.argtypes = [C.c_void_p]
        L.ref_ivox_dump.restype = C.c_size_t
        L.ref_ivox_dump.argtypes = [C.c_void_p, C.c_float, _i, _f, _i, C.c_size_t]
    if hasattr(L, "ref_ivox_set_nearby"):
        L.ref_ivox_set_nearby.argtypes = [C.c_void_p, C.c_int]
    L.ref_ivox_knn.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, C.c_double, _i, _f, _i, C.c_int]
    L.ref_ikd_create.restype = C.c_void_p
    L.ref_ikd_destroy.argtypes = [C.c_void_p]
    L.ref_ikd_build.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.ref_ikd_knn.argtypes = [C.c_void_p, _f, C.c_int, C.c_int, _i, _f, _i, C.c_int]
    if hasattr(L, "ref_ikd_delete_boxes"):
        L.ref_ikd_delete_boxes.restype = C.c_int
        L.ref_ikd_delete_boxes.argtypes = [C.c_void_p, _f, C.c_int]
    L.ref_esti_plane.argtypes = [_f, C.c_int, C.c_float, _f, _i]
    if hasattr(L, "ref_so3_exp"):
        L.ref_so3_exp.argtypes = [_d, C.c_double, _d]
    if hasattr(L, "ref_lio_hmodel"):
        L.ref_lio_hmodel.restype = C.c_int
        L.ref_lio_hmodel.argtypes = [C.c_void_p, _f, C.c_int, _d, _d, _d, _d, C.c_int, C.c_int, _f, _i, _i, _u8,
                                     _f, _f, _d, _d, _d, _i, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        L.ref_map_incremental.restype = C.c_int
        L.ref_map_incremental.argtypes = [C.c_void_p, _f, C.c_int, _d, _d, _d, _d, _f, _i, C.c_int, C.c_double, _f, _u8, C.c_int, C.c_int]
    return L


def _load_ref_reg():
    """The compiled reference matcher (oracle/ref_reg.cpp -> oracle/_ref/libref_reg.so)."""
    path = os.path.join(_HERE, "_ref", "libref_reg.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_reg_create.restype = C.c_void_p
    L.ref_reg_create.argtypes = [C.c_int, C.c_int]
    L.ref_reg_destroy.argtypes = [C.c_void_p]
    L.ref_reg_config.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double, C.c_int, C.c_longlong]
    L.ref_reg_set_source.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.ref_reg_set_target.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.ref_reg_align.restype = C.c_int
    L.ref_reg_align.argtypes = [C.c_void_p, _f, _f]
    L.ref_reg_fitness.restype = C.c_double
    L.ref_reg_fitness.argtypes = [C.c_void_p, C.c_double]
    if hasattr(L, "ref_calc_fitness_score"):
        L.ref_calc_fitness_score.restype = C.c_double
        L.ref_calc_fitness_score.argtypes = [_f, C.c_int, C.c_int, _f, C.c_int, C.c_int, _d, C.c_double]
    L.ref_reg_linearize.restype = C.c_double
    L.ref_reg_linearize.argtypes = [C.c_void_p, _d, C.c_void_p, C.c_void_p, C.c_void_p]
    L.ref_reg_compute_error.restype = C.c_double
    L.ref_reg_compute_error.argtypes = [C.c_void_p, _d]
    L.ref_reg_get_corr.argtypes = [C.c_void_p, _i]
    L.ref_reg_get_covs.argtypes = [C.c_void_p, C.c_int, _d]
    L.ref_vgicp_voxel.restype = C.c_int
    L.ref_vgicp_voxel.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _d, _d]
    L.ref_vgicp_coord.argtypes = [C.c_void_p, _d, _i]
    L.ref_se3_exp.argtypes = [_d, _d]
    return L


def _load_ref_cuda():
    """The compiled reference CUDA NDT (oracle/ref_cuda.cu -> oracle/_ref/libref_cuda.so).  Loading it needs the
    CUDA driver, so it is resolved lazily by the GPU tests / bench_extra (never at import time on a CPU box)."""
    path = os.path.join(_HERE, "_ref", "libref_cuda.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.refndt_create.restype = C.c_void_p
    L.refndt_create.argtypes = [C.c_double, C.c_int, C.c_int, C.c_double, C.c_double]
    L.refndt_destroy.argtypes = [C.c_void_p]
    L.refndt_set_source.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.refndt_set_target.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.refndt_num_voxels.restype = C.c_int
    L.refndt_num_voxels.argtypes = [C.c_void_p]
    L.refndt_num_correspondences.restype = C.c_int
    L.refndt_num_correspondences.argtypes = [C.c_void_p]
    L.refndt_linearize.restype = C.c_double
    L.refndt_linearize.argtypes = [C.c_void_p, _d, C.c_void_p, C.c_void_p]
    L.refndt_compute_error.restype = C.c_double
    L.refndt_compute_error.argtypes = [C.c_void_p, _d]
    L.refndt_align.restype = C.c_int
    L.refndt_align.argtypes = [C.c_void_p, _f, _f]
    return L


def _load_ref_cuda_vgicp():
    """The compiled reference CUDA VGICP (oracle/ref_cuda_vgicp.cu -> oracle/_ref/libref_cuda_vgicp.so); lazily, like
    _load_ref_cuda: loading it needs the CUDA driver."""
    path = os.path.join(_HERE, "_ref", "libref_cuda_vgicp.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.refvgicp_create.restype = C.c_void_p
    L.refvgicp_create.argtypes = [C.c_double, C.c_int, C.c_double, C.c_int]
    L.refvgicp_destroy.argtypes = [C.c_void_p]
    L.refvgicp_set_source.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.refvgicp_set_target.argtypes = [C.c_void_p, _f, C.c_int, C.c_int]
    L.refvgicp_linearize.restype = C.c_double
    L.refvgicp_linearize.argtypes = [C.c_void_p, _d, C.c_void_p, C.c_void_p]
    L.refvgicp_compute_error.restype = C.c_double
    L.refvgicp_compute_error.argtypes = [C.c_void_p, _d]
    L.refvgicp_align.restype = C.c_int
    L.refvgicp_align.argtypes = [C.c_void_p, _f, _f]
    return L


def _load_ref_ikfom():
    """The compiled reference filter + IMU stage (oracle/ref_ikfom.cpp -> oracle/_ref/libref_ikfom.so)."""
    path = os.path.join(_HERE, "_ref", "libref_ikfom.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_ikfom_predict.argtypes = [_d, _d, C.c_double, _d, _d, _d]
    L.ref_ikfom_update_rows.restype = C.c_int
    L.ref_ikfom_update_rows.argtypes = [_d, _d, _d, _d, _i, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, C.c_void_p]
    L.ref_ikfom_boxplus.argtypes = [_d, _d]
    L.ref_ikfom_boxminus.argtypes = [_d, _d, _d]
    L.ref_imu_create.restype = C.c_void_p
    L.ref_imu_create.argtypes = [_d, _d, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]
    L.ref_imu_destroy.argtypes = [C.c_void_p]
    L.ref_imu_process.restype = C.c_int
    L.ref_imu_process.argtypes = [C.c_void_p, _d, C.c_int, C.c_void_p, C.c_double, C.c_double, _f, _f, C.c_int, _d, _d, _f, _f]
    L.ref_imu_get_poses.restype = C.c_int
    L.ref_imu_get_poses.argtypes = [C.c_void_p, _d, C.c_int]
    L.ref_imu_is_init.restype = C.c_int
    L.ref_imu_is_init.argtypes = [C.c_void_p]
    return L


port = _load_port()
ref = _load_ref()
HAVE_REF = ref is not None
# the compiled iVox with a settable max_distance, explicit ids and the content dump (ref_lio.cpp's newer entry points)
HAVE_REF_IVOX_DUMP = HAVE_REF and hasattr(ref, "ref_ivox_dump")
ref_reg = _load_ref_reg()
HAVE_REF_REG = ref_reg is not None
ref_ikfom = _load_ref_ikfom()
HAVE_REF_IKFOM = ref_ikfom is not None


def _c32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


# ------------------------------------------------------------------ voxel grid
def voxelgrid(pts: np.ndarray, leaf: float = 0.5, want_vidx: bool = False):
    """PCL VoxelGrid restatement.  pts [n,4] -> [m,4] (ascending voxel index)."""
    pts = _c32(pts)
    n = pts.shape[0]
    out = np.empty((max(n, 1), 4), np.float32)
    vidx = np.empty(max(n, 1), np.int32)
    m = port.orc_voxelgrid(pts, n, leaf, out, vidx.ctypes.data)
    if m < 0:
        return (pts.copy(), None) if want_vidx else pts.copy()
    return (out[:m].copy(), vidx[:m].copy()) if want_vidx else out[:m].copy()


# ------------------------------------------------------------------ iVox (port)
class OracleIvox:
    """Restated faster_lio::IVox (ivox3d.h).  nearby in {0, 6, 18, 26, 74}."""

    def __init__(self, res: float = 0.5, nearby: int = 18, expected_cells: int = 1 << 16):
        self.h = port.orc_ivox_create(res, nearby, expected_cells)
        self.res = res

    def __del__(self):
        if getattr(self, "h", None):
            port.orc_ivox_destroy(self.h)
            self.h = None

    def set_nearby(self, nearby: int):
        port.orc_ivox_set_nearby(self.h, nearby)

    def add(self, xyz: np.ndarray, id0: int):
        xyz = _c32(xyz)
        port.orc_ivox_add(self.h, xyz, xyz.shape[1], xyz.shape[0], id0, None)

    @property
    def num_cells(self):
        return port.orc_ivox_num_cells(self.h)

    def delete_boxes(self, boxes: np.ndarray) -> int:
        """KD_TREE::Delete_Point_Boxes semantics on the hash map: min <= p < max per axis."""
        b = _c32(np.asarray(boxes).reshape(-1, 6))
        return int(port.orc_ivox_delete_boxes(self.h, b, b.shape[0]))

    @property
    def num_points(self):
        return port.orc_ivox_num_points(self.h)

    def knn(self, q: np.ndarray, k: int = 5, max_sq: float = 5.0, exact: bool = False, nthreads: int = 8, reference_order: bool = False):
        """-> ids [nq,k] (-1 pad), d2 [nq,k] (-1 pad), xyz [nq,k,3], cnt [nq]; canonical (d2,id) order, or with
        reference_order the order IVox::GetClosestPoint leaves its output in (libstdc++'s nth_element, ivox3d.h:159-164)."""
        q = _c32(q)
        nq = q.shape[0]
        ids = np.empty((nq, k), np.int32)
        d2 = np.empty((nq, k), np.float32)
        xyz = np.empty((nq, k, 3), np.float32)
        cnt = np.empty(nq, np.int32)
        assert not (exact and reference_order)
        port.orc_knn(self.h, 1 if exact else 2 if reference_order else 0, q, q.shape[1], nq, k, max_sq, ids, d2, xyz, cnt, nthreads)
        return ids, d2, xyz, cnt


def esti_plane(pts5: np.ndarray, thr: float = 0.1):
    pts5 = _c32(pts5).reshape(-1, 5, 3)
    n = pts5.shape[0]
    pabcd = np.empty((n, 4), np.float32)
    ok = np.empty(n, np.int32)
    port.orc_esti_plane_batch(pts5, n, thr, pabcd, ok)
    return pabcd, ok


# ------------------------------------------------------------------ compiled reference
class RefIvox:
    """The reference's own faster_lio::IVox, compiled unmodified (oracle/_ref)."""

    def __init__(self, res: float = 0.5, nearby: int = 18, capacity: int = 1 << 30, max_distance: float = 100.0):
        assert HAVE_REF, "oracle/_ref/libref_lio.so not built"
        # an older library hard-wires max_distance = 100 (the extra argument is then ignored)
        assert HAVE_REF_IVOX_DUMP or max_distance == 100.0, "oracle/_ref/libref_lio.so predates ref_ivox_create's max_distance"
        self.res = res
        self.h = ref.ref_ivox_create(res, nearby, capacity, float(max_distance))

    def __del__(self):
        if getattr(self, "h", None):
            ref.ref_ivox_destroy(self.h)
            self.h = None

    def add(self, xyz: np.ndarray, id0: int, distance: float = 0.0):
        """IVox::AddPoints(points, distance): `distance` = travel_distance, what the LRU ages voxels by (ivox3d.h:251)."""
        xyz = _c32(xyz[:, :3])
        ref.ref_ivox_add(self.h, xyz, xyz.shape[0], id0, float(distance))

    def add_ids(self, xyz: np.ndarray, ids: np.ndarray, distance: float = 0.0):
        """AddPoints with an explicit id per point."""
        xyz = _c32(xyz[:, :3])
        ids = np.ascontiguousarray(ids, np.int32)
        assert ids.shape == (xyz.shape[0],)
        ref.ref_ivox_add_ids(self.h, xyz, ids, xyz.shape[0], float(distance))

    def set_nearby(self, nearby: int):
        ref.ref_ivox_set_nearby(self.h, nearby)

    @property
    def num_cells(self):
        return ref.ref_ivox_num_cells(self.h)

    @property
    def num_points(self):
        return ref.ref_ivox_num_points(self.h)

    def dump(self):
        """-> keys [n,3] int32, xyz [n,3] float32, ids [n] int32: every stored point (IVox::GetAllPoints), each voxel's
        points in insertion order; keys are computed by Pos2Grid's expression in C++ (Eigen rounds half away from zero)."""
        n = ref.ref_ivox_num_points(self.h)
        keys = np.empty((max(n, 1), 3), np.int32)
        xyz = np.empty((max(n, 1), 3), np.float32)
        ids = np.empty(max(n, 1), np.int32)
        m = ref.ref_ivox_dump(self.h, self.res, keys, xyz, ids, n)
        assert m == n
        return keys[:n], xyz[:n], ids[:n]

    def knn(self, q: np.ndarray, k: int = 5, max_sq: float = 5.0, nthreads: int = 8):
        """-> ids [nq,k], xyz [nq,k,3], cnt [nq] in the REFERENCE's order (nearest first)."""
        q = _c32(q[:, :3])
        nq = q.shape[0]
        ids = np.empty((nq, k), np.int32)
        xyz = np.empty((nq, k, 3), np.float32)
        cnt = np.empty(nq, np.int32)
        ref.ref_ivox_knn(self.h, q, nq, k, max_sq, ids, xyz, cnt, nthreads)
        return ids, xyz, cnt


class RefIkd:
    """The reference's ikd-Tree (KD_TREE<PointXYZINormal>), compiled unmodified."""

    def __init__(self):
        assert HAVE_REF
        self.h = ref.ref_ikd_create()

    def __del__(self):
        if getattr(self, "h", None):
            ref.ref_ikd_destroy(self.h)
            self.h = None

    def build(self, xyz: np.ndarray, id0: int = 0):
        xyz = _c32(xyz[:, :3])
        ref.ref_ikd_build(self.h, xyz, xyz.shape[0], id0)

    def delete_boxes(self, boxes: np.ndarray) -> int:
        b = _c32(np.asarray(boxes).reshape(-1, 6))
        return ref.ref_ikd_delete_boxes(self.h, b, b.shape[0])

    def knn(self, q: np.ndarray, k: int = 5, nthreads: int = 8):
        q = _c32(q[:, :3])
        nq = q.shape[0]
        ids = np.empty((nq, k), np.int32)
        d2 = np.empty((nq, k), np.float32)
        cnt = np.empty(nq, np.int32)
        ref.ref_ikd_knn(self.h, q, nq, k, ids, d2, cnt, nthreads)
        return ids, d2, cnt


def ref_esti_plane(pts5: np.ndarray, thr: float = 0.1):
    assert HAVE_REF
    pts5 = _c32(pts5).reshape(-1, 5, 3)
    n = pts5.shape[0]
    pabcd = np.empty((n, 4), np.float32)
    ok = np.empty(n, np.int32)
    ref.ref_esti_plane(pts5, n, thr, pabcd, ok)
    return pabcd, ok


def _qr_call(L, name, pts5):
    pts5 = _c32(pts5).reshape(-1, 5, 3)
    n = pts5.shape[0]
    qr = np.empty((n, 15), np.float32); hc = np.empty((n, 3), np.float32); perm = np.empty((n, 3), np.int32)
    nz = np.empty(n, np.int32); x = np.empty((n, 3), np.float32)
    fn = getattr(L, name)
    fn.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
    fn.restype = None
    fn(pts5.ctypes.data, n, qr.ctypes.data, hc.ctypes.data, perm.ctypes.data, nz.ctypes.data, x.ctypes.data)
    return dict(qr=qr, hcoeffs=hc, perm=perm, nonzero_pivots=nz, x=x)


def esti_plane_qr(pts5: np.ndarray):
    """The port's factorisation behind esti_plane with its intermediates (packed QR column-major, Householder coefficients,
    column permutation, non-zero pivots, solution)."""
    return _qr_call(port, "orc_esti_plane_qr", pts5)


def ref_esti_plane_qr(pts5: np.ndarray):
    """The same intermediates from Eigen's ColPivHouseholderQR as esti_plane instantiates it (oracle/ref_lio.cpp)."""
    assert HAVE_REF and hasattr(ref, "ref_esti_plane_qr")
    return _qr_call(ref, "ref_esti_plane_qr", pts5)


def canonical_rows(ids: np.ndarray, d2: np.ndarray):
    """Sort each k-NN row ascending by (d2, id) with -1 padding last (the repo-wide canonical order)."""
    big = np.where(ids < 0, np.inf, d2.astype(np.float64))
    idk = np.where(ids < 0, np.iinfo(np.int32).max, ids)
    key = np.empty(ids.shape, dtype=[("d", np.float64), ("i", np.int64)])
    key["d"] = big
    key["i"] = idk
    order = np.argsort(key, axis=1, order=("d", "i"), kind="stable")
    return np.take_along_axis(ids, order, 1), np.take_along_axis(d2, order, 1)
