"""TEST INFRASTRUCTURE ONLY — CPU restatement of the scan matcher.

* Levenberg-Marquardt on SE(3): fast_gicp::LsqRegistration
  (slam/thirdparty/fast_gicp/include/fast_gicp/gicp/impl/lsq_registration_impl.hpp:71-131,163-208),
  se3_exp (include/fast_gicp/so3/so3.hpp:60-104) — numpy, written independently of csrc/reg.cu.
* cost functions: oracle/lsd_oracle.c (orc_ndt_cost, orc_gicp_cost, orc_fitness).
Pin status: the GICP / VGICP cost functions, the covariances, se3_exp and the whole LM loop are checked
against the COMPILED reference classes (oracle/ref_reg.cpp -> oracle/_ref/libref_reg.so: the reference's
own LsqRegistration / FastGICP / FastVGICP headers, with our PCL/Boost shims) in tests/test_oracle_reg.py.
NDT (P2D): the reference NDT exists only as CUDA code; its own sources recompile for sm_90a
(oracle/ref_cuda.cu -> oracle/_ref/libref_cuda.so, RefNdtCuda below) and pin the NDT restatement and the product's
NDT kernels on the GPU box (tests/test_gpu_ref_cuda.py).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import oracle as O


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0.0]])


def so3_exp_quat(omega):
    th2 = float(omega @ omega)
    if th2 < 1e-10:
        tq = th2 * th2
        imag = 0.5 - th2 / 48.0 + tq / 3840.0
        real = 1.0 - th2 / 8.0 + tq / 384.0
    else:
        th = np.sqrt(th2)
        imag = np.sin(0.5 * th) / th
        real = np.cos(0.5 * th)
    return np.array([imag * omega[0], imag * omega[1], imag * omega[2], real])


def se3_exp(a):
    from .eskf import quat_to_R
    omega = a[:3]
    theta = np.sqrt(omega @ omega)
    R = quat_to_R(so3_exp_quat(omega))
    Om = skew(omega)
    if theta < 1e-10:
        V = R
    else:
        V = np.eye(3) + (1 - np.cos(theta)) / theta ** 2 * Om + (theta - np.sin(theta)) / theta ** 3 * (Om @ Om)
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = V @ a[3:]
    return T


def rot_angle_deg(R):
    c = np.clip((np.trace(R) - 1) / 2, -1, 1)
    s = np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
    return np.degrees(np.arctan2(s, c))


class OracleMatcher:
    """kind 'ndt' (P2D), 'gicp' or 'vgicp'.  Protocol of pcl::Registration."""

    def __init__(self, kind="ndt", resolution=1.0, neighbors=7, max_iterations=64, trans_eps=0.01, rot_eps=None, k=20,
                 max_corr=2.0, map_res=0.5, normal_sq=25.0, nthreads=8):
        self.kind, self.res, self.nb, self.max_it = kind, resolution, neighbors, max_iterations
        self.trans_eps = trans_eps
        self.rot_eps = rot_eps if rot_eps is not None else (0.1 if kind == "ndt" else 1e-2)
        self.k, self.max_corr, self.map_res, self.normal_sq, self.nthreads = k, max_corr, map_res, normal_sq, nthreads
        self.lm_max, self.lm_init = 10, 1e-9
        self.ndt = None
        self.tmap = None
        self.vg = None

    def __del__(self):
        if getattr(self, "ndt", None):
            O.port.orc_ndt_destroy(self.ndt)
        if getattr(self, "vg", None):
            O.port.orc_vgicp_destroy(self.vg)

    def _normals(self, pts):
        m = O.OracleIvox(self.map_res, 18, max(pts.shape[0], 1024))
        m.add(np.ascontiguousarray(pts[:, :3]), 0)
        nrm = np.zeros((pts.shape[0], 3))
        cnt = np.zeros(pts.shape[0], np.int32)
        O.port.orc_gicp_normals(m.h, pts, pts.shape[1], pts.shape[0], self.k, self.normal_sq, nrm, cnt, self.nthreads)
        return m, nrm

    def set_target(self, pts):
        self.tgt = np.ascontiguousarray(pts, np.float32)
        if self.kind == "ndt":
            if self.ndt:
                O.port.orc_ndt_destroy(self.ndt)
            self.ndt = O.port.orc_ndt_build(self.tgt, self.tgt.shape[1], self.tgt.shape[0], self.res)
            self.n_voxels = O.port.orc_ndt_num_voxels(self.ndt)
        else:
            self.tmap, self.tgt_nrm = self._normals(self.tgt)
            if self.kind == "vgicp":
                if self.vg:
                    O.port.orc_vgicp_destroy(self.vg)
                self.vg = O.port.orc_vgicp_build(self.tgt, self.tgt.shape[1], self.tgt.shape[0], self.tgt_nrm, float(self.res))
                self.n_voxels = O.port.orc_vgicp_num_voxels(self.vg)

    def set_source(self, pts):
        self.src = np.ascontiguousarray(pts, np.float32)
        n = self.src.shape[0]
        if self.kind == "gicp":
            _, self.src_nrm = self._normals(self.src)
            self.corr = np.full(n, -1, np.int32)
            self.maha = np.zeros((n, 9))
        elif self.kind == "vgicp":
            _, self.src_nrm = self._normals(self.src)
            self.vcorr = np.full(self.nb * n, -1, np.int64)
            self.vmaha = np.zeros((self.nb * n, 9))

    def cost(self, T, update=True, deriv=True):
        T = np.ascontiguousarray(T, np.float64)
        H, b = np.zeros(36), np.zeros(6)
        Hp = H.ctypes.data if deriv else None
        bp = b.ctypes.data if deriv else None
        if self.kind == "ndt":
            if update:
                self.T_lin = T.copy()
            nc = C.c_int()
            e = O.port.orc_ndt_cost(self.ndt, self.src, self.src.shape[1], self.src.shape[0], self.T_lin, T, self.nb, Hp, bp, C.byref(nc))
            self.n_corr = nc.value
        elif self.kind == "vgicp":
            nc = C.c_int()
            e = O.port.orc_vgicp_cost(self.vg, self.src, self.src.shape[1], self.src_nrm, self.src.shape[0], T, self.nb, int(update),
                                      self.vcorr, self.vmaha, Hp, bp, C.byref(nc))
            self.n_corr = nc.value
        else:
            e = O.port.orc_gicp_cost(self.tmap.h, self.tgt, self.tgt.shape[1], self.tgt_nrm, self.src, self.src.shape[1], self.src_nrm,
                                     self.src.shape[0], T, self.max_corr, int(update), self.corr, self.maha, Hp, bp, self.nthreads)
            self.n_corr = int((self.corr >= 0).sum())
        return e, H.reshape(6, 6), b

    def _conv(self, delta, scale=1.0):
        r = rot_angle_deg(delta[:3, :3]) / (self.rot_eps * scale)
        t = np.abs(delta[:3, 3]).max() / (self.trans_eps * scale)
        return max(r, t) < 1

    def align(self, guess):
        x0 = np.array(guess, np.float64)
        lam = -1.0
        self.converged = False
        self.iterations = 0
        for it in range(self.max_it):
            if self.converged:
                break
            self.iterations = it
            y0, H, b = self.cost(x0, True, True)
            if lam < 0:
                lam = self.lm_init * np.abs(np.diag(H)).max()
            nu = 2.0
            stepped = False
            for _ in range(self.lm_max):
                try:
                    d = np.linalg.solve(H + lam * np.eye(6), -b)
                except np.linalg.LinAlgError:   # LDLT of a singular system: the reference would produce NaNs and give up
                    break
                delta = se3_exp(d)
                xi = delta @ x0
                yi, _, _ = self.cost(xi, False, False)
                rho = (y0 - yi) / (d @ (lam * d - b))
                if rho < 0:
                    if self._conv(delta, 10.0):
                        stepped = True
                        break
                    lam = nu * lam
                    nu = 2 * nu
                    continue
                x0 = xi
                lam = lam * max(1.0 / 3.0, 1 - (2 * rho - 1) ** 3)
                stepped = True
                break
            if not stepped:
                break
            self.converged = self._conv(delta)
        self.final = x0
        return x0

    def fitness(self, T=None, max_range=25.0):
        """getFitnessScore(max_range): the mean fp32 squared distance from each source point (transformed in fp32) to its
        nearest target point, over the points where it is <= max_range, however far that neighbour is.  Ranges up to 64
        map voxels go through the grid search of orc_fitness, longer ones through a scan of the whole target."""
        T = np.ascontiguousarray(self.final if T is None else T, np.float64)
        if max_range > 64.0 * self.map_res * self.map_res * 64.0:
            return _fitness_scan(self.tgt, self.src, T, max_range)
        if self.tmap is None:
            self.tmap = O.OracleIvox(self.map_res, 18, max(self.tgt.shape[0], 1024))
            self.tmap.add(np.ascontiguousarray(self.tgt[:, :3]), 0)
        return O.port.orc_fitness(self.tmap.h, self.src, self.src.shape[1], self.src.shape[0], T, max_range, max_range)


def _fitness_scan(tgt, src, T, max_range, chunk=256):
    """orc_fitness by a scan of the whole target: the same fp32 transform ((r0 x + r1 y) + r2 z) + t and fp32 squared
    distance (dx dx + dy dy) + dz dz, the float d2 compared with the double max_range, the sum in double in source order."""
    R, t = T[:3, :3].astype(np.float32), T[:3, 3].astype(np.float32)
    a = np.ascontiguousarray(src[:, :3], np.float32)
    q = np.stack([R[r, 0] * a[:, 0] + R[r, 1] * a[:, 1] + R[r, 2] * a[:, 2] + t[r] for r in range(3)], 1)
    P = np.ascontiguousarray(tgt[:, :3], np.float32)
    best = np.empty(len(q), np.float32)
    for i in range(0, len(q), chunk):
        d = P[None, :, :] - q[i:i + chunk, None, :]
        best[i:i + chunk] = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).min(1)
    s, nr = 0.0, 0
    for v in best.astype(np.float64):
        if v <= max_range:
            s += v
            nr += 1
    return s / nr if nr > 0 else 1.7976931348623157e308


class RefMatcher:
    """The COMPILED reference matcher (fast_gicp::FastGICP / FastVGICP through oracle/_ref/libref_reg.so)."""

    def __init__(self, kind="gicp", resolution=1.0, neighbors=1, max_iterations=64, trans_eps=0.01, rot_eps=1e-2, k=20,
                 max_corr=2.0, nthreads=1, max_process_time_us=0):
        if not O.HAVE_REF_REG:
            raise RuntimeError("oracle/_ref/libref_reg.so missing (built only where /root/reference exists)")
        self.kind = kind
        self.h = O.ref_reg.ref_reg_create(1 if kind == "gicp" else 2, nthreads)
        O.ref_reg.ref_reg_config(self.h, max_iterations, trans_eps, rot_eps, max_corr if kind == "gicp" else -1.0, k, resolution,
                                 neighbors, max_process_time_us)

    def __del__(self):
        if getattr(self, "h", None):
            O.ref_reg.ref_reg_destroy(self.h)
            self.h = None

    def set_target(self, pts):
        self.tgt = np.ascontiguousarray(pts, np.float32)
        O.ref_reg.ref_reg_set_target(self.h, self.tgt, self.tgt.shape[0], self.tgt.shape[1])

    def set_source(self, pts):
        self.src = np.ascontiguousarray(pts, np.float32)
        O.ref_reg.ref_reg_set_source(self.h, self.src, self.src.shape[0], self.src.shape[1])

    def covs(self, which):
        n = (self.tgt if which else self.src).shape[0]
        out = np.zeros((n, 9))
        O.ref_reg.ref_reg_get_covs(self.h, int(which), out)
        return out.reshape(n, 3, 3)

    def linearize(self, T, deriv=True):
        T = np.ascontiguousarray(T, np.float64)
        H, b = np.zeros(36), np.zeros(6)
        nc = C.c_int()
        e = O.ref_reg.ref_reg_linearize(self.h, T, H.ctypes.data if deriv else None, b.ctypes.data if deriv else None, C.byref(nc))
        self.n_corr = nc.value
        return e, H.reshape(6, 6), b

    def compute_error(self, T):
        return O.ref_reg.ref_reg_compute_error(self.h, np.ascontiguousarray(T, np.float64))

    def corr(self):
        out = np.zeros(self.src.shape[0], np.int32)
        O.ref_reg.ref_reg_get_corr(self.h, out)
        return out

    def align(self, guess):
        out = np.zeros(16, np.float32)
        self.converged = bool(O.ref_reg.ref_reg_align(self.h, np.ascontiguousarray(guess, np.float32).reshape(16), out))
        return out.reshape(4, 4).astype(np.float64)

    def fitness(self, max_range=25.0):
        return O.ref_reg.ref_reg_fitness(self.h, float(max_range))

    def voxel(self, x, y, z):
        mean, cov = np.zeros(3), np.zeros(9)
        n = O.ref_reg.ref_vgicp_voxel(self.h, int(x), int(y), int(z), mean, cov)
        return n, mean, cov.reshape(3, 3)

    def coord(self, p):
        c = np.zeros(3, np.int32)
        O.ref_reg.ref_vgicp_coord(self.h, np.ascontiguousarray(p, np.float64), c)
        return c


def ref_calc_fitness_score(tgt, src, T, max_range):
    """InformationMatrixCalculator::calc_fitness_score (information_matrix_calculator.cpp:71-102) COMPILED from the reference:
    the in-tree twin of pcl::Registration::getFitnessScore."""
    tgt = np.ascontiguousarray(tgt, np.float32); src = np.ascontiguousarray(src, np.float32)
    return O.ref_reg.ref_calc_fitness_score(tgt, tgt.shape[0], tgt.shape[1], src, src.shape[0], src.shape[1],
                                            np.ascontiguousarray(T, np.float64), float(max_range))


def ref_se3_exp(a):
    T = np.zeros(16)
    O.ref_reg.ref_se3_exp(np.ascontiguousarray(a, np.float64), T)
    return T.reshape(4, 4)


class RefNdtCuda:
    """The COMPILED reference CUDA NDT (fast_gicp::NDTCuda over NDTCudaCore), sm_90a build; needs a GPU."""
    _lib = None

    def __init__(self, resolution=1.0, neighbors=7, max_iterations=64, trans_eps=0.01, rot_eps=0.1):
        if RefNdtCuda._lib is None:
            RefNdtCuda._lib = O._load_ref_cuda()
        if RefNdtCuda._lib is None:
            raise RuntimeError("oracle/_ref/libref_cuda.so missing (built only where /root/reference exists)")
        self.L = RefNdtCuda._lib
        self.h = self.L.refndt_create(resolution, neighbors, max_iterations, trans_eps, rot_eps)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.refndt_destroy(self.h)
            self.h = None

    def set_target(self, pts):
        self.tgt = np.ascontiguousarray(pts, np.float32)
        self.L.refndt_set_target(self.h, self.tgt, self.tgt.shape[0], self.tgt.shape[1])
        self.n_voxels = self.L.refndt_num_voxels(self.h)

    def set_source(self, pts):
        self.src = np.ascontiguousarray(pts, np.float32)
        self.L.refndt_set_source(self.h, self.src, self.src.shape[0], self.src.shape[1])

    def linearize(self, T, deriv=True):
        T = np.ascontiguousarray(T, np.float64)
        H, b = np.zeros(36), np.zeros(6)
        e = self.L.refndt_linearize(self.h, T, H.ctypes.data if deriv else None, b.ctypes.data if deriv else None)
        self.n_corr = self.L.refndt_num_correspondences(self.h)
        return e, H.reshape(6, 6), b

    def compute_error(self, T):
        return self.L.refndt_compute_error(self.h, np.ascontiguousarray(T, np.float64))

    def align(self, guess):
        out = np.zeros(16, np.float32)
        self.converged = bool(self.L.refndt_align(self.h, np.ascontiguousarray(guess, np.float32).reshape(16), out))
        return out.reshape(4, 4).astype(np.float64)


class RefVgicpCuda:
    """The COMPILED reference CUDA VGICP (fast_gicp::FastVGICPCuda over FastVGICPCudaCore), sm_90a build; needs a GPU.
    Parameters of registrations.cpp:43-55 ("FAST_VGICP_CUDA"): resolution 1.0, eps 0.01, 64 iterations, k = 20, source /
    target neighbours from a CPU k-d tree (nn_method 0), DIRECT1 voxel correspondences."""
    _lib = None

    def __init__(self, resolution=1.0, max_iterations=64, trans_eps=0.01, nn_method=0):
        if RefVgicpCuda._lib is None:
            RefVgicpCuda._lib = O._load_ref_cuda_vgicp()
        if RefVgicpCuda._lib is None:
            raise RuntimeError("oracle/_ref/libref_cuda_vgicp.so missing (built only where /root/reference exists)")
        self.L = RefVgicpCuda._lib
        self.h = self.L.refvgicp_create(resolution, max_iterations, trans_eps, nn_method)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.refvgicp_destroy(self.h)
            self.h = None

    def set_target(self, pts):
        self.tgt = np.ascontiguousarray(pts, np.float32)
        self.L.refvgicp_set_target(self.h, self.tgt, self.tgt.shape[0], self.tgt.shape[1])

    def set_source(self, pts):
        self.src = np.ascontiguousarray(pts, np.float32)
        self.L.refvgicp_set_source(self.h, self.src, self.src.shape[0], self.src.shape[1])

    def linearize(self, T, deriv=True):
        T = np.ascontiguousarray(T, np.float64)
        H, b = np.zeros(36), np.zeros(6)
        e = self.L.refvgicp_linearize(self.h, T, H.ctypes.data if deriv else None, b.ctypes.data if deriv else None)
        return e, H.reshape(6, 6), b

    def compute_error(self, T):
        return self.L.refvgicp_compute_error(self.h, np.ascontiguousarray(T, np.float64))

    def align(self, guess):
        out = np.zeros(16, np.float32)
        self.converged = bool(self.L.refvgicp_align(self.h, np.ascontiguousarray(guess, np.float32).reshape(16), out))
        return out.reshape(4, 4).astype(np.float64)
