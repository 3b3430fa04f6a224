"""CPU restatement of OverlapDetector (slam/localization/include/overlap_merge.hpp:38-304), the overlap detector that
MapLoader::mergeMapSLAM (map_loader.cpp:118-137) runs over fragments of 10 new key frames when both maps share a GNSS origin.

The scan matching is oracle.reg.OracleMatcher: "ndt" for the coarse stage (NDT_CUDA), "gicp" with max_corr = 0.5 and
transformation epsilon 0.001 for the finetune (FAST_GICP).  Plain numpy / scipy otherwise; written from the reference's
statements, not from the device code.  pcl::transformPointCloud with a double matrix is taken to evaluate each row
((r0 x + r1 y) + r2 z) + t in double and round to float (unpinned against PCL, which is not in the reference tree).
"""
from __future__ import annotations

from collections import deque

import numpy as np

DBL_MAX = np.finfo(np.float64).max
F = np.float32

DEFAULTS = dict(distance_thresh=30.0, candidate_link_dist=10, max_candidate_num=3, fitness_score_max_range=25.0,
                fitness_score_thresh=1.5, fitness_inlier_thresh=0.2)
FILTER_RANGE, FILTER_MIN_Z, INLIER_MAX_RANGE = F(100.0), F(0.5), 1.0


def connections(edges) -> dict:
    """connection_map (:80-91): id -> set of ids, both directions."""
    m: dict = {}
    for a, b in edges:
        m.setdefault(int(a), set()).add(int(b))
        m.setdefault(int(b), set()).add(int(a))
    return m


def connection_count(conn, source, target, max_count) -> int:
    """get_connection_count (:265-296) as written: a FIFO queue, visited marked when a node is popped, levels counted."""
    visited = {k: False for k in conn}
    q = deque([source])
    count = 0
    while q:
        for _ in range(len(q)):
            curr = q.popleft()
            if curr == target:
                return count
            visited[curr] = True
            for adj in sorted(conn.get(curr, ())):
                if not visited.get(adj, False):
                    q.append(adj)
        count += 1
        if max_count > 0 and count >= max_count:
            break
    return count


def knn10(poses, keyframes, new_slot):
    """nearestKSearch(k = 10) over the key frames' translations as float points: float squared distances
    ((dx dx + dy dy) + dz dz); equal distances in keyframes order.  Returns [(d2, slot)]."""
    q = np.asarray(poses[new_slot][:3, 3], F)
    hits = []
    for pos, k in enumerate(keyframes):
        d = np.asarray(poses[k][:3, 3], F) - q
        d2 = F(F(F(d[0] * d[0]) + F(d[1] * d[1])) + F(d[2] * d[2]))
        hits.append((d2, pos, int(k)))
    hits.sort(key=lambda h: (h[0], h[1]))
    return [(h[0], h[2]) for h in hits[:10]]


def find_candidates(poses, ids, keyframes, new_slot, edges, **kw) -> list[int]:
    """find_candidates (:113-145): slots."""
    p = dict(DEFAULTS, **kw)
    conn = connections(edges)
    new_id = ids[new_slot]
    out = []
    for d2, k in knn10(poses, keyframes, new_slot):
        if ids[k] == new_id:
            continue
        if ids[k] in conn.get(new_id, set()):
            continue
        if float(d2) < p["distance_thresh"] * p["distance_thresh"]:
            if connection_count(conn, new_id, ids[k], p["candidate_link_dist"]) >= p["candidate_link_dist"]:
                out.append(k)
        if len(out) >= p["max_candidate_num"]:
            break
    return out


def _sum3(a, b, c):
    return (a + b) + c


def iso_inverse(T):
    """Eigen Isometry inverse: R^T, -(R^T t), each sum left to right (dtype of T)."""
    R, t = T[:3, :3], T[:3, 3]
    G = np.eye(4, dtype=T.dtype)
    G[:3, :3] = R.T
    for a in range(3):
        G[a, 3] = -_sum3(R[0, a] * t[0], R[1, a] * t[1], R[2, a] * t[2])
    return G


def iso_mul(A, B):
    """Isometry product: R_a R_b, R_a t_b + t_a, each sum left to right."""
    G = np.eye(4, dtype=A.dtype)
    for a in range(3):
        for b in range(3):
            G[a, b] = _sum3(A[a, 0] * B[0, b], A[a, 1] * B[1, b], A[a, 2] * B[2, b])
        G[a, 3] = _sum3(A[a, 0] * B[0, 3], A[a, 1] * B[1, 3], A[a, 2] * B[2, 3]) + A[a, 3]
    return G


def guess(T_new, T_cand) -> np.ndarray:
    """(new->mOdom.inverse() * cand->mOdom).matrix().cast<float>() (:159)."""
    return iso_mul(iso_inverse(np.asarray(T_new, np.float64)), np.asarray(T_cand, np.float64)).astype(F)


def finetune_guess(ndt_final) -> np.ndarray:
    """Eigen::Isometry3f(relative_pose).inverse().matrix() (:198), in float."""
    M = np.asarray(ndt_final, F).copy()
    M[3] = (0, 0, 0, 1)
    return iso_inverse(M)


def filt(pts) -> np.ndarray:
    """filter() (:213-223): sqrtf(x*x + y*y) < 100 and z > 0.5, in float."""
    x, y, z = (np.asarray(pts[:, i], F) for i in range(3))
    r = np.sqrt((x * x + y * y).astype(F)).astype(F)
    return pts[(r < FILTER_RANGE) & (z > FILTER_MIN_Z)]


def transform_f(pts, T) -> np.ndarray:
    """pcl::transformPointCloud with a Matrix4f: ((r0 x + r1 y) + r2 z) + t in float."""
    T = np.asarray(T, F)
    a = np.asarray(pts[:, :3], F)
    out = np.array(pts, F, copy=True)
    for r in range(3):
        out[:, r] = ((T[r, 0] * a[:, 0] + T[r, 1] * a[:, 1]) + T[r, 2] * a[:, 2]) + T[r, 3]
    return out


def transform_d(pts, T) -> np.ndarray:
    """pcl::transformPointCloud with a Matrix4d: ((r0 x + r1 y) + r2 z) + t in double, stored as float."""
    T = np.asarray(T, np.float64)
    a = np.asarray(pts[:, :3], np.float64)
    out = np.array(pts, F, copy=True)
    for r in range(3):
        out[:, r] = (((T[r, 0] * a[:, 0] + T[r, 1] * a[:, 1]) + T[r, 2] * a[:, 2]) + T[r, 3]).astype(F)
    return out


def nn_d2(tgt, q, chunk=512) -> np.ndarray:
    """Exact float squared distance ((dx dx + dy dy) + dz dz) of every query to its nearest target point (brute force)."""
    P = np.ascontiguousarray(tgt[:, :3], F)
    out = np.empty(len(q), F)
    for i in range(0, len(q), chunk):
        d = P[None, :, :] - q[i:i + chunk, None, :3]
        out[i:i + chunk] = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).min(1)
    return out


def calc_fitness_score(cloud1, cloud2, T, max_range):
    """calc_fitness_score(target = cloud1, source = cloud2, relpose, max_range) (:225-263): (score, ratio, nr, n_filtered)."""
    tgt = filt(np.asarray(cloud1, F))
    src = filt(transform_f(cloud2, T))
    if len(src) == 0 or len(tgt) == 0:
        return DBL_MAX, 0.0, 0, len(src)
    d2 = nn_d2(tgt, np.asarray(src[:, :3], F)).astype(np.float64)
    ok = d2 <= max_range
    nr = int(ok.sum())
    if nr == 0:
        return DBL_MAX, 0.0, 0, len(src)
    return float(d2[ok].sum() / nr), nr / len(src), nr, len(src)


def accumulate(clouds, poses, ids, keyframes, edges, best):
    """accum_points (:186-194), with keyframe_id_map's default 0 for an id outside keyframes."""
    conn = connections(edges)
    id_index = {}
    for i, k in enumerate(keyframes):
        id_index[ids[k]] = i
    parts = [np.asarray(clouds[best], F)]
    inv = iso_inverse(np.asarray(poses[best], np.float64))
    for c in sorted(conn.get(ids[best], ())):
        k = keyframes[id_index.get(c, 0)]
        parts.append(transform_d(clouds[k], iso_mul(inv, np.asarray(poses[k], np.float64))))
    return np.concatenate(parts, 0)


class OracleOverlapDetector:
    """OverlapDetector::detect over clouds[slot] (sensor frame) with graph ids ids[slot]."""

    def __init__(self, clouds, ids, **kw):
        self.clouds, self.ids = clouds, ids
        self.p = dict(DEFAULTS, **kw)

    def matching(self, cands, new_slot, poses, keyframes, edges):
        from oracle.reg import OracleMatcher
        rep = dict(new_slot=new_slot, n_candidates=len(cands), candidates=list(cands), n_prescreened=0, best_slot=-1,
                   best_score=DBL_MAX, n_accum=0)
        if not cands:
            return rep, None, "no_candidates"
        reg = OracleMatcher("ndt")
        reg.set_target(self.clouds[new_slot])
        best_score, best, rel = DBL_MAX, None, None
        for k in cands:
            g = guess(poses[new_slot], poses[k])
            if calc_fitness_score(self.clouds[new_slot], self.clouds[k], g, INLIER_MAX_RANGE)[1] < self.p["fitness_inlier_thresh"]:
                continue
            rep["n_prescreened"] += 1
            reg.set_source(self.clouds[k])
            T = reg.align(g.astype(np.float64))
            if not reg.converged:
                continue
            score = reg.fitness(T=T, max_range=self.p["fitness_score_max_range"])
            if score > best_score:
                continue
            best_score, best, rel = score, k, T.astype(F)
        if best is None:
            return rep, None, "no_match"
        rep.update(best_slot=best, best_score=best_score)
        accum = accumulate(self.clouds, poses, self.ids, keyframes, edges, best)
        rep["n_accum"] = len(accum)
        acc = OracleMatcher("gicp", max_corr=0.5, trans_eps=0.001)
        acc.set_target(accum)
        acc.set_source(self.clouds[new_slot])
        T = acc.align(finetune_guess(rel).astype(np.float64))
        if not acc.converged:
            return rep, None, "gicp_diverged"
        relpose = T.astype(F)
        score = calc_fitness_score(accum, self.clouds[new_slot], relpose, self.p["fitness_score_max_range"])[0]
        rep["score"] = score
        if score > self.p["fitness_score_thresh"]:
            return rep, None, "gicp_reject"
        return rep, dict(key1=best, key2=new_slot, relpose=relpose.astype(np.float64), score=score, coarse_score=best_score), "found"

    def detect(self, poses, keyframes, new_keyframes, edges):
        overlaps, reports = [], []
        for ns in new_keyframes:
            cands = find_candidates(poses, self.ids, keyframes, ns, edges, **self.p)
            rep, ov, decision = self.matching(cands, ns, poses, keyframes, edges)
            rep["decision"] = decision
            reports.append(rep)
            if ov is not None:
                overlaps.append(ov)
        return overlaps, reports
