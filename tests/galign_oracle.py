"""CPU restatement of the closure search of global_alignment (slam/localization/include/global_alignment.hpp:200-258).

Made of the reference's own pieces where they exist as compiled code: SCManager (makeScancontext at the nine search_trans
offsets, buildRingKeyKDTree, detectCandidateMatch) from oracle/_ref/libref_keyframe.so, FastVGICP from oracle/_ref/libref_reg.so
(oracle.reg.RefMatcher), and getFitnessScore as oracle/lsd_oracle.c's orc_fitness.  The merge of the candidate lists per
database index (std::map<int, SCMatch>, :207-227) and yaw2matrix (Scancontext.cpp:68-75) are restated here in Python,
written from the reference's statements, not from the device code.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

SEARCH_TRANS = [(0, 0), (-4, 0), (4, 0), (0, -4), (0, 4), (-4, -4), (-4, 4), (4, -4), (4, 4)]   # :210-212
SC_DIST_THRES, ICP_SCORE_THRES, FITNESS_SCORE_MAX = 0.30, 1.5, 25.0                             # :31-34

_REF_KF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_keyframe.so")
HAVE_REF = os.path.exists(_REF_KF) and os.path.exists(os.path.join(os.path.dirname(_REF_KF), "libref_reg.so"))


def shift_to_yaw(shift) -> np.float32:
    """deg2rad(float) of shift * PC_UNIT_SECTORANGLE (Scancontext.cpp:356; Scancontext.h: 360 / 60 degrees)."""
    deg = np.float32(float(shift) * (360.0 / 60.0))
    return np.float32(float(deg) * math.pi / 180.0)


def candidates_from_query(idx, dist, shift, n_cand, thres=SC_DIST_THRES):
    """detectCandidateMatch's filter (Scancontext.cpp:346-358) over one offset's ring-key candidates, in candidate order:
    [(sc_idx, sc_yaw float32, sc_dist float32)] for dist < thres."""
    return [(int(idx[c]), shift_to_yaw(shift[c]), np.float32(dist[c])) for c in range(int(n_cand)) if dist[c] < thres]


def merge_candidates(per_offset):
    """:207-227: for each offset in order, each candidate in order, matches[sc_idx] = match when it is new or its float
    sc_dist is strictly smaller.  Returns [(sc_idx, sc_dist, sc_yaw)] in ascending sc_idx (std::map order)."""
    matches = {}
    for cands in per_offset:
        for idx, yaw, dist in cands:
            if idx not in matches or matches[idx][0] > dist:
                matches[idx] = (np.float32(dist), np.float32(yaw))
    return [(k, matches[k][0], matches[k][1]) for k in sorted(matches)]


def yaw2matrix(y) -> np.ndarray:
    """Eigen::Matrix4f with cos / sin of the float y, returned as double."""
    c, s = np.float32(math.cos(float(np.float32(y)))), np.float32(math.sin(float(np.float32(y))))
    T = np.eye(4, dtype=np.float32)
    T[0, 0], T[0, 1], T[1, 0], T[1, 1] = c, -s, s, c
    return T.astype(np.float64)


def orc_fitness(tgt, src, T, max_range=FITNESS_SCORE_MAX, map_res=0.5):
    """getFitnessScore(max_range) of src at T (applied in float) against tgt: oracle/lsd_oracle.c's orc_fitness."""
    from oracle import oracle as O
    m = O.OracleIvox(map_res, 18, max(tgt.shape[0], 1024))
    m.add(np.ascontiguousarray(tgt[:, :3]), 0)
    src = np.ascontiguousarray(src, np.float32)
    return O.port.orc_fitness(m.h, src, src.shape[1], src.shape[0], np.ascontiguousarray(T, np.float64), float(max_range),
                              min(float(max_range), 64.0 * map_res * map_res * 64.0))


class OracleGlobalAlignment:
    """The search loop of global_alignment over reference clouds (the database, in order) and new clouds."""

    def __init__(self, ref_clouds):
        self.L = C.CDLL(_REF_KF)
        _pd, _pf, _pi = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int)
        self.L.ref_sc_make.argtypes = [_pf, C.c_int, C.c_double, C.c_double, _pd, _pd, _pd]
        self.L.ref_sc_make.restype = None
        self.L.ref_sc_db_create.argtypes = [_pd, C.c_int, C.c_double]
        self.L.ref_sc_db_create.restype = C.c_void_p
        self.L.ref_sc_db_destroy.argtypes = [C.c_void_p]
        self.L.ref_sc_detect_candidates.argtypes = [C.c_void_p, _pd, _pi, _pf, _pf, C.c_int]
        self.L.ref_sc_detect_candidates.restype = C.c_int
        self.refs = [np.ascontiguousarray(c, np.float32) for c in ref_clouds]
        descs = np.stack([self.make(c, 0.0, 0.0) for c in self.refs])   # KeyFrame's descriptor (keyframe.cpp:165-167)
        self.db = self.L.ref_sc_db_create(descs.ctypes.data_as(_pd), len(self.refs), SC_DIST_THRES)

    def __del__(self):
        if getattr(self, "db", None):
            self.L.ref_sc_db_destroy(self.db)
            self.db = None

    def make(self, cloud, dx, dy):
        cloud = np.ascontiguousarray(cloud, np.float32)
        d, rk, sk = np.zeros(1200), np.zeros(20), np.zeros(60)
        p = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
        self.L.ref_sc_make(p(cloud, C.c_float), cloud.shape[0], dx, dy, p(d, C.c_double), p(rk, C.c_double), p(sk, C.c_double))
        return d

    def matches(self, cloud):
        """:209-227 for one new key frame: [(sc_idx, sc_dist, sc_yaw)], ascending sc_idx."""
        per_offset = []
        for dx, dy in SEARCH_TRANS:
            d = self.make(cloud, float(dx), float(dy))
            idx, yaw, dist = np.zeros(10, np.int32), np.zeros(10, np.float32), np.zeros(10, np.float32)
            n = self.L.ref_sc_detect_candidates(self.db, d.ctypes.data_as(C.POINTER(C.c_double)), idx.ctypes.data_as(C.POINTER(C.c_int)),
                                                yaw.ctypes.data_as(C.POINTER(C.c_float)), dist.ctypes.data_as(C.POINTER(C.c_float)), 10)
            per_offset.append([(int(idx[i]), yaw[i], dist[i]) for i in range(n)])
        return merge_candidates(per_offset)

    def search(self, new_clouds):
        """:206-258: closures [dict(ref, new, relpose float32, score, sc_dist, sc_yaw)] in new-key-frame order, then ascending
        reference index; and every pair tried."""
        from oracle.reg import RefMatcher
        closures, tried = [], []
        for q, cloud in enumerate(new_clouds):
            cloud = np.ascontiguousarray(cloud, np.float32)
            for ref, dist, yaw in self.matches(cloud):
                reg = RefMatcher("vgicp", resolution=1.0, neighbors=1, max_iterations=64, trans_eps=0.1, rot_eps=0.1, k=20)
                reg.set_target(self.refs[ref])
                reg.set_source(cloud)
                T = reg.align(yaw2matrix(-yaw))
                rec = dict(ref=ref, new=q, sc_dist=dist, sc_yaw=yaw, converged=reg.converged, relpose=T.astype(np.float32))
                tried.append(rec)
                if not reg.converged:
                    continue
                rec["score"] = orc_fitness(self.refs[ref], cloud, T)
                if rec["score"] < ICP_SCORE_THRES:
                    closures.append(rec)
        return closures, tried
