"""CPU restatement of hdl_graph_slam::LoopDetector (loop_detector.hpp:33-231) and of the fitness / weight of
InformationMatrixCalculator (information_matrix_calculator.cpp:25-47,71-102, weight() in the header :44-47).

The scan matching is oracle.reg.OracleMatcher: "ndt" for the coarse stage (NDT_CUDA), "gicp" with max_corr = 0.5 for the
refinement (FAST_GICP).  Plain numpy / scipy otherwise; written from the reference's statements, not from the device code.
"""
from __future__ import annotations

import math

import numpy as np

DBL_MAX = np.finfo(np.float64).max

DEFAULTS = dict(distance_thresh=15.0, accum_distance_thresh=25.0, distance_from_last_edge_thresh=15.0,
                distance_new_keyframe_thresh=2.0, distance_keyframe_thresh=2.0, fitness_score_max_range=25.0,
                fitness_score_thresh=1.5)


def normalized_rotation(R) -> np.ndarray:
    """Eigen::Quaterniond(R).normalized().toRotationMatrix()"""
    m = lambda i, j: float(R[i][j])  # noqa: E731
    q = [0.0, 0.0, 0.0, 0.0]  # x y z w
    t = m(0, 0) + m(1, 1) + m(2, 2)
    if t > 0:
        s = math.sqrt(t + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[0], q[1], q[2] = (m(2, 1) - m(1, 2)) * s, (m(0, 2) - m(2, 0)) * s, (m(1, 0) - m(0, 1)) * s
    else:
        i = 0
        if m(1, 1) > m(0, 0):
            i = 1
        if m(2, 2) > m(i, i):
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3] = (m(k, j) - m(j, k)) * s
        q[j] = (m(j, i) + m(i, j)) * s
        q[k] = (m(k, i) + m(i, k)) * s
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    x, y, z, w = (v / n for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def initial_guess(T_new, T_cand) -> np.ndarray:
    """matching() :165-173: both rotations normalised, new^-1 * candidate in double, cast to float, (2,3) zeroed."""
    Rn, Rc = normalized_rotation(T_new[:3, :3]), normalized_rotation(T_cand[:3, :3])
    G = np.eye(4)
    G[:3, :3] = Rn.T @ Rc
    G[:3, 3] = Rn.T @ (np.asarray(T_cand[:3, 3]) - np.asarray(T_new[:3, 3]))
    G = G.astype(np.float32).astype(np.float64)
    G[2, 3] = 0.0
    return G


def find_candidates(poses, accum, keyframes, new_slot, last_edge_accum_distance=0.0, **kw):
    p = dict(DEFAULTS, **kw)
    if accum[new_slot] - last_edge_accum_distance < p["distance_from_last_edge_thresh"]:
        return []
    out = []
    acc_kf = -100.0
    for k in keyframes:
        if accum[new_slot] - accum[k] < p["accum_distance_thresh"]:
            continue
        if accum[k] - acc_kf < p["distance_keyframe_thresh"]:
            continue
        d = poses[k][:2, 3] - poses[new_slot][:2, 3]
        if math.sqrt(d[0] * d[0] + d[1] * d[1]) > p["distance_thresh"]:
            continue
        acc_kf = accum[k]
        out.append(int(k))
    return out


def weight(a, max_x, min_y, max_y, x):
    y = (1.0 - math.exp(-a * x)) / (1.0 - math.exp(-a * max_x))
    return min_y + (max_y - min_y) * y


def information_matrix(fitness_score) -> np.ndarray:
    """calc_information_matrix with the constructor's constants; w_x / w_q are floats in the reference."""
    w_x = float(np.float32(weight(20.0, 0.5, 0.1 ** 2, 5.0 ** 2, fitness_score)))
    w_q = float(np.float32(weight(20.0, 0.5, 0.05 ** 2, 0.2 ** 2, fitness_score)))
    inf = np.eye(6)
    inf[:3, :3] /= w_x
    inf[3:, 3:] /= w_q
    return inf


def calc_fitness_score(tgt, src, T, max_range=DBL_MAX):
    """Mean squared 1-NN distance of the (float-)transformed source points to the target, those <= max_range."""
    from scipy.spatial import cKDTree
    Tf = np.asarray(T, np.float32)
    s = np.asarray(src[:, :3], np.float32)
    q = (s @ Tf[:3, :3].T + Tf[:3, 3]).astype(np.float32)
    t = np.asarray(tgt[:, :3], np.float32)
    _, idx = cKDTree(t.astype(np.float64)).query(q.astype(np.float64), k=1)
    d = t[idx] - q
    d2 = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float64)
    ok = d2 <= max_range
    return (float(d2[ok].sum() / ok.sum()) if ok.any() else DBL_MAX), int(ok.sum())


class OracleLoopDetector:
    """LoopDetector::detect over clouds[slot] (sensor frame) with accum[slot]."""

    def __init__(self, clouds, accum, **kw):
        self.clouds, self.accum = clouds, accum
        self.p = dict(DEFAULTS, **kw)
        self.last_edge_accum_distance = 0.0

    def matching(self, cands, new_slot, poses):
        from oracle.reg import OracleMatcher
        rep = dict(new_slot=new_slot, n_candidates=len(cands), best_slot=-1, best_score=DBL_MAX, candidates=list(cands))
        reg = OracleMatcher("ndt")
        reg.set_target(self.clouds[new_slot])
        best_score, best, rel = DBL_MAX, None, None
        for k in cands:
            reg.set_source(self.clouds[k])
            T = reg.align(initial_guess(poses[new_slot], poses[k]))
            if not reg.converged:
                continue
            score = reg.fitness(T=T, max_range=self.p["fitness_score_max_range"])
            if score > best_score:
                continue
            best_score, best, rel = score, k, T.astype(np.float32)
        rep.update(best_slot=-1 if best is None else best, best_score=best_score)
        if best_score > 2.0 * self.p["fitness_score_thresh"]:
            return rep, None, "coarse_reject"
        acc = OracleMatcher("gicp", max_corr=0.5)
        acc.set_target(self.clouds[new_slot])
        acc.set_source(self.clouds[best])
        T = acc.align(rel.astype(np.float64))
        if not acc.converged:
            return rep, None, "gicp_diverged"
        score = acc.fitness(T=T, max_range=self.p["fitness_score_max_range"])
        if score > self.p["fitness_score_thresh"]:
            return rep, None, "gicp_reject"
        self.last_edge_accum_distance = self.accum[new_slot]
        relpose = T.astype(np.float32)
        fit, _ = calc_fitness_score(self.clouds[new_slot], self.clouds[best], relpose)
        loop = dict(key1=new_slot, key2=best, relpose=relpose, coarse_score=best_score, score=score,
                    information=information_matrix(fit), fitness=fit, n_candidates=len(cands))
        return rep, loop, "found"

    def detect(self, poses, keyframes, new_keyframes):
        loops, reports = [], []
        acc_new = 0.0
        for ns in new_keyframes:
            if self.accum[ns] - acc_new < self.p["distance_new_keyframe_thresh"]:
                reports.append(dict(new_slot=ns, decision="skipped"))
                continue
            acc_new = self.accum[ns]
            cands = find_candidates(poses, self.accum, keyframes, ns, self.last_edge_accum_distance,
                                    **{k: self.p[k] for k in DEFAULTS})
            if not cands:
                reports.append(dict(new_slot=ns, decision="no_candidates", n_candidates=0))
                continue
            rep, loop, decision = self.matching(cands, ns, poses)
            rep["decision"] = decision
            reports.append(rep)
            if loop is not None:
                loops.append(loop)
        return loops, reports
