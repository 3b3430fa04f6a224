"""TEST INFRASTRUCTURE ONLY — numpy restatement of the detection voxelizer.

Follows sensor_driver/inference/voxelize (relative to /root/reference):
  preprocess_kernel.cu:6-20,56-101   sliding window, 3x4 motion, time + 0.1
  voxelization_kernel.cu:73-180      hash voxelisation, <= max_points_per_voxel points, mean, fp16
executed SEQUENTIALLY in point order (the reference's GPU result depends on thread arrival order;
the sequential order is one of its possible outcomes).  Pin status: the reference has no CPU implementation of this
path, but its two .cu files recompile unmodified for sm_90a (oracle/ref_vfe.cu -> oracle/_ref/libref_vfe.so, class
RefVoxelizer below) and pin this restatement's semantics and the product on the GPU box (tests/test_gpu_ref_cuda.py).
Where the product deviates from the reference on purpose (include/lsdreg.h), this follows the product: the row counted for
an empty realtime frame is FAR_ROW_XYZ, and the window transform carries every feature past z (time + 0.1 only when
num_feature > 4).
"""
from __future__ import annotations

import numpy as np

# The row lsd_vfe_accumulate counts for an empty realtime frame (the reference counts one row there and copies it from
# the caller's empty array): finite, and far enough out that no rigid motion brings it into a range box.
FAR_ROW_XYZ = 1e30


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded, on arrays.  a*b is exact in float64; TwoSum gives s + e == a*b + c exactly,
    and s rounds to the fp32 nearest a*b + c unless s is itself halfway between two floats, where e breaks the tie."""
    a64, b64, c64 = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a64 * b64
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        r = s.astype(np.float32)
        other = np.nextafter(r, np.where(s > r.astype(np.float64), np.float32(np.inf), np.float32(-np.inf)))
        mid = s == (r.astype(np.float64) + other.astype(np.float64)) * 0.5
        to_other = mid & np.isfinite(s) & (e != 0) & ~np.isnan(e) & ((e > 0) == (other > r))
    return np.where(to_other, other, r).astype(np.float32)


class OracleVoxelizer:
    def __init__(self, min_range=(-64, -64, -2), max_range=(64, 64, 4), voxel_size=(0.1, 0.1, 0.15), max_ppv=5,
                 max_voxels=300000, max_points=500000, nf=5, max_frames=2):
        self.mn = np.array(min_range, np.float32)
        self.mx = np.array(max_range, np.float32)
        self.vs = np.array(voxel_size, np.float32)
        self.gs = np.round((self.mx - self.mn) / self.vs).astype(np.int64)
        self.max_ppv, self.max_voxels, self.max_points, self.nf = max_ppv, max_voxels, max_points, nf
        self.frame_pts = [0] * max_frames
        self.total = 0
        self.buf = np.zeros((0, nf), np.float32)

    def accumulate(self, pts, motion=None, realtime=True):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, self.nf)
        n = pts.shape[0]
        if realtime:
            m = np.ascontiguousarray(np.eye(4) if motion is None else motion, np.float32).ravel()
            self.total -= self.frame_pts[-1]
            n = max(min(n, self.max_points - self.total), 1)
            if pts.shape[0] == 0:                                    # the one counted row of an empty frame
                pts = np.zeros((1, self.nf), np.float32)
                pts[0, :3] = FAR_ROW_XYZ
            self.frame_pts = [0] + self.frame_pts[:-1]
            old = self.buf[:self.total]
            out = old.copy()                                         # features 3.. carried over
            if self.total > 0:
                with np.errstate(invalid="ignore", over="ignore"):
                    for r in range(3):  # as nvcc contracts the reference's m0*x + m1*y + m2*z + m3 (SASS of transform_kernel:
                        # FMUL m1*y; FFMA m0*x + .; FFMA m2*z + .; FADD m3), each step rounded to fp32
                        t = m[4 * r + 1] * old[:, 1]
                        t = fma32(m[4 * r], old[:, 0], t)
                        t = fma32(m[4 * r + 2], old[:, 2], t)
                        out[:, r] = t + m[4 * r + 3]
                    if self.nf > 4:                                  # the time channel
                        out[:, 4] = (old[:, 4].astype(np.float64) + 0.1).astype(np.float32)
            self.buf = np.concatenate([pts[:n], out], 0)
        else:
            self.frame_pts = [0] * len(self.frame_pts)
            self.total = 0
            n = min(n, self.max_points)
            self.buf = pts[:n].copy()
        self.frame_pts[0] = n
        self.total += n
        return self.total

    def cells(self, points):
        """Per point: its cell (x, y, z) = floor((p - min) / voxel_size) in fp32, whether it passes the range test
        (min <= p < max per axis) and whether its cell lies in the grid.  NaN on an axis passes the range test and
        lands in cell 0 of that axis: the comparisons are false and the device's float-to-int conversion gives 0."""
        p = np.ascontiguousarray(points, np.float32)
        ijk = np.zeros((p.shape[0], 3), np.int64)
        in_range = np.ones(p.shape[0], bool)
        in_grid = np.ones(p.shape[0], bool)
        for a in range(3):
            c = p[:, a]
            with np.errstate(invalid="ignore", over="ignore"):
                q = np.floor((c - self.mn[a]) / self.vs[a])
            q = np.where(np.isnan(q), 0.0, np.clip(q, -1.0, float(self.gs[a])))
            ijk[:, a] = q.astype(np.int64)
            in_range &= ((c >= self.mn[a]) & (c < self.mx[a])) | np.isnan(c)
            in_grid &= (ijk[:, a] >= 0) & (ijk[:, a] < self.gs[a])
        return ijk, in_range, in_grid

    def voxelize(self, points=None, zyx=True):
        p = self.buf[:self.total] if points is None else np.ascontiguousarray(points, np.float32)
        ijk, in_range, in_grid = self.cells(p)
        inr = in_range & in_grid
        ids = np.nonzero(inr)[0]
        off = (ijk[ids, 2] * self.gs[1] + ijk[ids, 1]) * self.gs[0] + ijk[ids, 0]
        uniq, first, inv, cnt = np.unique(off, return_index=True, return_inverse=True, return_counts=True)
        vorder = np.argsort(first, kind="stable")            # voxel ids in order of first point
        vid_of_uniq = np.empty_like(vorder); vid_of_uniq[vorder] = np.arange(len(vorder))
        V = min(len(uniq), self.max_voxels)
        srt = np.lexsort((ids, vid_of_uniq[inv]))             # points grouped by voxel id, ascending index inside
        gv = vid_of_uniq[inv][srt]
        start = np.searchsorted(gv, np.arange(len(uniq)))
        feat = np.zeros((V, self.nf), np.float32)
        npts = np.minimum(cnt[vorder][:V], self.max_ppv).astype(np.uint32)
        with np.errstate(invalid="ignore", over="ignore"):
            for k in range(self.max_ppv):
                has = npts > k
                src = ids[srt[start[:V][has] + k]]
                if k == 0:
                    feat[has] = p[src]
                else:
                    feat[has] = feat[has] + p[src]            # fp32, sequential order
            feat = (feat / npts[:, None].astype(np.float32)).astype(np.float16)
        firstpt = ids[first[vorder][:V]]
        idx = np.zeros((V, 4), np.uint32)
        c = ijk[firstpt]
        idx[:, 1:] = c[:, ::-1] if zyx else c
        return feat, idx, npts


class RefVoxelizer:
    """The COMPILED reference voxelizer (Preprocess + Voxelization kernels recompiled for sm_90a:
    oracle/ref_vfe.cu -> oracle/_ref/libref_vfe.so).  Needs a GPU; loaded lazily."""
    _lib = None

    def __init__(self, min_range=(-64.0, -64.0, -2.0), max_range=(64.0, 64.0, 4.0), voxel_size=(0.1, 0.1, 0.15), max_points_per_voxel=5,
                 max_voxels=300000, max_points=500000, num_feature=5, max_frame_num=2):
        import ctypes as C
        import os
        if RefVoxelizer._lib is None:
            path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libref_vfe.so")
            if not os.path.exists(path):
                raise RuntimeError("oracle/_ref/libref_vfe.so missing (built only where /root/reference exists)")
            L = C.CDLL(path)
            f32 = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
            L.refvfe_create.restype = C.c_void_p
            L.refvfe_create.argtypes = [f32, f32, f32, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
            L.refvfe_destroy.argtypes = [C.c_void_p]
            L.refvfe_accumulate.restype = C.c_int
            L.refvfe_accumulate.argtypes = [C.c_void_p, f32, C.c_int, f32, C.c_int]
            L.refvfe_get_points.restype = C.c_int
            L.refvfe_get_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
            L.refvfe_voxelize.restype = C.c_int
            L.refvfe_voxelize.argtypes = [C.c_void_p, C.c_int]
            L.refvfe_get_output.restype = C.c_int
            L.refvfe_get_output.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
            RefVoxelizer._lib = L
        self.L = RefVoxelizer._lib
        self.nf = num_feature
        self.h = self.L.refvfe_create(np.asarray(min_range, np.float32), np.asarray(max_range, np.float32), np.asarray(voxel_size, np.float32),
                                      max_points_per_voxel, max_voxels, max_points, num_feature, max_frame_num)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.refvfe_destroy(self.h)
            self.h = None

    def accumulate(self, points, motion=None, realtime=True):
        pts = np.ascontiguousarray(points, np.float32)
        m = np.ascontiguousarray(np.eye(4) if motion is None else motion, np.float32)
        return self.L.refvfe_accumulate(self.h, pts, pts.shape[0], m.reshape(-1), int(realtime))

    def points(self):
        n = self.L.refvfe_get_points(self.h, None, 0)
        out = np.empty((n, self.nf), np.float32)
        self.L.refvfe_get_points(self.h, out.ctypes.data, n)
        return out

    def voxelize(self, zyx=True):
        v = self.L.refvfe_voxelize(self.h, int(zyx))
        feat = np.empty((v, self.nf), np.float16)
        idx = np.empty((v, 4), np.uint32)
        self.L.refvfe_get_output(self.h, feat.ctypes.data, idx.ctypes.data)
        return feat, idx
