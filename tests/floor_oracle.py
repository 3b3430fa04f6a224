"""CPU restatement of floor detection (FloorDetectionNodelet::detect after PrefilteringNodelet, and the detect_ground copies)
in the PCL 1.9.1 / Boost semantics DESIGN.md section 5f states: the rules lsd_floor_* runs on the device, written out in numpy
so the GPU suite can compare every stage.

- prefilter: the C oracle's pcl::VoxelGrid (oracle.voxelgrid), then d > near && d < far with d = double(float |xyz|);
- clip: two PlaneClipper3D passes with planes (0, 0, 1, d), in float;
- normals: the exact 10 nearest in (fp32 d2, index) order, computeMeanAndCovarianceMatrix in float, pcl::eigen33,
  flipNormalTowardsViewpoint, and normal_filtering's double(|normalized(n).z|) > cos(deg);
- RANSAC: boost::mt19937 seeded 12345, drawIndexSample, isSampleGood, computeModelCoefficients, countWithinDistance and the
  stop rule of RandomSampleConsensus::computeModel, then selectWithinDistance of the best model.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.spatial import cKDTree

F = np.float32
MAPPING, GROUND, RENDER = 0, 1, 2
FOUND, EMPTY, FEW_CANDIDATES, NO_MODEL, FEW_INLIERS, NOT_VERTICAL = range(6)


def default_params(preset: int) -> dict:
    p = dict(prefilter_leaf=0.0, distance_near=0.1, distance_far=100.0, clip_keep_d=1.5, clip_cut_d=-1.5,
             use_normal_filtering=1, normal_filter_deg=20.0, viewpoint_z=0.0, ransac_threshold=0.1, ransac_probability=0.99,
             ransac_max_iterations=10000, floor_pts_thresh=1024, floor_normal_deg=10.0)
    if preset == MAPPING:
        p.update(prefilter_leaf=0.2, clip_keep_d=2.0, clip_cut_d=-1.0)
    elif preset == RENDER:
        p.update(ransac_threshold=0.2)
    return p


# ------------------------------------------------------------------ generator
class MT19937:
    """boost::mt19937 / std::mt19937: init_genrand seeding, the standard twist and tempering."""

    def __init__(self, seed: int = 12345):
        mt = [seed & 0xffffffff]
        for i in range(1, 624):
            mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + i) & 0xffffffff)
        self.mt = np.array(mt, np.uint32)
        self.buf = np.zeros(0, np.uint32)
        self.pos = 0

    def _twist(self):
        mt = self.mt
        up, lo, a = np.uint32(0x80000000), np.uint32(0x7fffffff), np.uint32(0x9908b0df)

        def upd(i0, i1):   # entries i0 .. i1-1 together: each reads mt[i + 1] (old) and mt[i + 397 mod 624] (final)
            i = np.arange(i0, i1)
            y = (mt[i] & up) | (mt[(i + 1) % 624] & lo)
            mt[i] = mt[(i + 397) % 624] ^ (y >> np.uint32(1)) ^ np.where((y & np.uint32(1)) != 0, a, np.uint32(0))
        upd(0, 227)
        upd(227, 454)
        upd(454, 623)
        upd(623, 624)
        y = mt.copy()
        y ^= y >> np.uint32(11)
        y ^= (y << np.uint32(7)) & np.uint32(0x9d2c5680)
        y ^= (y << np.uint32(15)) & np.uint32(0xefc60000)
        y ^= y >> np.uint32(18)
        self.buf = y
        self.pos = 0

    def next(self) -> int:
        if self.pos >= self.buf.size:
            self._twist()
        v = int(self.buf[self.pos])
        self.pos += 1
        return v

    def outputs(self, n: int) -> np.ndarray:
        out = np.empty(n, np.uint32)
        k = 0
        while k < n:
            if self.pos >= self.buf.size:
                self._twist()
            m = min(n - k, self.buf.size - self.pos)
            out[k:k + m] = self.buf[self.pos:self.pos + m]
            self.pos += m
            k += m
        return out


# ------------------------------------------------------------------ stages
def prefilter(pts: np.ndarray, p: dict) -> np.ndarray:
    from oracle import oracle
    # pcl::VoxelGrid skips non-finite points of a cloud that is not dense (the C oracle's grid assumes a dense cloud)
    fin = np.isfinite(pts[:, :3]).all(axis=1)
    v = oracle.voxelgrid(pts[fin], p["prefilter_leaf"])
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    d = np.sqrt((x * x + y * y) + z * z).astype(np.float64)
    return v[(d > p["distance_near"]) & (d < p["distance_far"])]


def clip_mask(pts: np.ndarray, p: dict) -> np.ndarray:
    with np.errstate(invalid="ignore"):
        h = (F(0) * pts[:, 0] + F(0) * pts[:, 1]) + F(1) * pts[:, 2]
        return (h >= -F(p["clip_keep_d"])) & ~(h >= -F(p["clip_cut_d"]))


def knn10(xyz: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """The exact 10 nearest of every point (itself included) in (fp32 d2, index) order: [n,10] indices (-1 pad), counts."""
    n = xyz.shape[0]
    k = min(10, n)
    nbr = np.full((n, 10), -1, np.int64)
    if n == 0:
        return nbr, np.zeros(0, np.int64)
    tree = cKDTree(xyz.astype(np.float64))
    kq = min(n, 16)
    dist, idx = tree.query(xyz.astype(np.float64), k=kq)
    dist = dist.reshape(n, kq); idx = idx.reshape(n, kq)

    def d2(i, js):
        d = xyz[js] - xyz[i]
        return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]

    # rows whose 16-candidate list surely holds the fp32 top 10: the k-th float64 distance is clearly below the last one
    safe = (kq == n) | (dist[:, k - 1] * (1 + 1e-5) + 1e-12 < dist[:, kq - 1])
    rows = np.nonzero(safe)[0]
    if rows.size:
        cand = idx[rows]
        dd = d2(rows[:, None], cand)
        key = np.argsort(cand, axis=1, kind="stable")   # by index, then stably by d2: (d2, index) order
        cand = np.take_along_axis(cand, key, 1); dd = np.take_along_axis(dd, key, 1)
        o2 = np.argsort(dd, axis=1, kind="stable")
        nbr[rows, :k] = np.take_along_axis(cand, o2, 1)[:, :k]
    for i in np.nonzero(~safe)[0]:
        r = dist[i, k - 1] * (1 + 1e-4) + 1e-9
        js = np.array(sorted(tree.query_ball_point(xyz[i].astype(np.float64), r)), np.int64)
        dd = d2(i, js)
        o = np.lexsort((js, dd))
        nbr[i, :k] = js[o][:k]
    return nbr, np.full(n, k, np.int64)


def _roots2(b, c):
    d = ((b * b).astype(np.float64) - 4.0 * c.astype(np.float64)).astype(F)
    d = np.where(d < 0, F(0), d)
    sd = np.sqrt(d)
    return np.zeros_like(b), F(0.5) * (b - sd), F(0.5) * (b + sd)


def eigen33(C: np.ndarray):
    """pcl::eigen33 (smallest eigenvalue and its vector) of [n,9] float32 matrices, vectorised."""
    scale = np.abs(C).max(axis=1)
    scale = np.where(scale <= np.finfo(F).tiny, F(1), scale).astype(F)
    S = (C / scale[:, None]).astype(F)
    m00, m01, m02, m11, m12, m22 = S[:, 0], S[:, 1], S[:, 2], S[:, 4], S[:, 5], S[:, 8]
    c0 = m00 * m11 * m22 + F(2) * m01 * m02 * m12 - m00 * m12 * m12 - m11 * m02 * m02 - m22 * m01 * m01
    c1 = m00 * m11 - m01 * m01 + m00 * m22 - m02 * m02 + m11 * m22 - m12 * m12
    c2 = m00 + m11 + m22
    with np.errstate(invalid="ignore", divide="ignore"):
        s_inv3, s_sqrt3 = F(1.0 / 3.0), np.sqrt(F(3))
        c2o3 = c2 * s_inv3
        a3 = (c1 - c2 * c2o3) * s_inv3
        a3 = np.where(a3 > 0, F(0), a3)
        hb = F(0.5) * (c0 + c2o3 * (F(2) * c2o3 * c2o3 - c1))
        q = hb * hb + a3 * a3 * a3
        q = np.where(q > 0, F(0), q)
        rho = np.sqrt(-a3)
        th = np.arctan2(np.sqrt(-q), hb) * s_inv3
        ct, st = np.cos(th), np.sin(th)
        r = np.stack([c2o3 + F(2) * rho * ct, c2o3 - rho * (ct + s_sqrt3 * st), c2o3 - rho * (ct - s_sqrt3 * st)], 1).astype(F)
        # the sort of computeRoots: swap(0, 1) if r0 >= r1; if r1 >= r2 { swap(1, 2); swap(0, 1) if r0 >= r1 }

        def swap(a, b, sw):
            ra, rb = r[:, a].copy(), r[:, b].copy()
            r[:, a] = np.where(sw, rb, ra); r[:, b] = np.where(sw, ra, rb)
        swap(0, 1, r[:, 0] >= r[:, 1])
        second = r[:, 1] >= r[:, 2]
        swap(1, 2, second)
        swap(0, 1, second & (r[:, 0] >= r[:, 1]))
        quad = (np.abs(c0) < np.finfo(F).eps) | (r[:, 0] <= 0)
        q0, q1, q2 = _roots2(c2, c1)
        r0 = np.where(quad, q0, r[:, 0])
    lam = r0 * scale
    S = S.copy()
    for j in (0, 4, 8):
        S[:, j] = S[:, j] - r0
    R0, R1, R2 = S[:, 0:3], S[:, 3:6], S[:, 6:9]

    def cross(a, b):
        return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                         a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    v1, v2, v3 = cross(R0, R1), cross(R0, R2), cross(R1, R2)
    sq = lambda v: (v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]  # noqa: E731
    l1, l2, l3 = sq(v1), sq(v2), sq(v3)
    pick1 = (l1 >= l2) & (l1 >= l3)
    pick2 = ~pick1 & (l2 >= l1) & (l2 >= l3)
    v = np.where(pick1[:, None], v1, np.where(pick2[:, None], v2, v3))
    l = np.where(pick1, l1, np.where(pick2, l2, l3))
    with np.errstate(invalid="ignore", divide="ignore"):
        v = v / np.sqrt(l)[:, None]
    return lam.astype(F), v.astype(F)


def normals(xyz: np.ndarray, vpz: float = 0.0):
    """NormalEstimation (k = 10) of the clipped cloud: normal4 [n,4] (after the viewpoint flip), cov6 [n,6], neighbours."""
    n = xyz.shape[0]
    nbr, cnt = knn10(xyz)
    k = min(10, n)
    acc = np.zeros((n, 9), F)
    for r in range(k):
        q = xyz[nbr[:, r]]
        x, y, z = q[:, 0], q[:, 1], q[:, 2]
        acc[:, 0] += x * x; acc[:, 1] += x * y; acc[:, 2] += x * z
        acc[:, 3] += y * y; acc[:, 4] += y * z; acc[:, 5] += z * z
        acc[:, 6] += x; acc[:, 7] += y; acc[:, 8] += z
    acc = (acc / F(max(k, 1))).astype(F)
    C = np.zeros((n, 9), F)
    C[:, 0] = acc[:, 0] - acc[:, 6] * acc[:, 6]; C[:, 1] = acc[:, 1] - acc[:, 6] * acc[:, 7]; C[:, 2] = acc[:, 2] - acc[:, 6] * acc[:, 8]
    C[:, 4] = acc[:, 3] - acc[:, 7] * acc[:, 7]; C[:, 5] = acc[:, 4] - acc[:, 7] * acc[:, 8]; C[:, 8] = acc[:, 5] - acc[:, 8] * acc[:, 8]
    C[:, 3] = C[:, 1]; C[:, 6] = C[:, 2]; C[:, 7] = C[:, 5]
    lam, v = eigen33(C)
    es = (C[:, 0] + C[:, 4]) + C[:, 8]
    with np.errstate(invalid="ignore", divide="ignore"):
        curv = np.where(es != 0, np.abs(lam / es), F(0)).astype(F)
    vp = np.stack([F(0) - xyz[:, 0], F(0) - xyz[:, 1], F(vpz) - xyz[:, 2]], 1)
    cos_t = (vp[:, 0] * v[:, 0] + vp[:, 1] * v[:, 1]) + vp[:, 2] * v[:, 2]
    v = np.where((cos_t < 0)[:, None], v * F(-1), v)
    nrm = np.concatenate([v, curv[:, None]], 1).astype(F)
    cov6 = C[:, [0, 1, 2, 4, 5, 8]].copy()
    if k < 3:
        nrm[:] = np.nan; cov6[:] = np.nan
    return nrm, cov6, nbr


def normal_nz(nrm: np.ndarray) -> np.ndarray:
    """normalized(n).z in float (Eigen: n / sqrt(squaredNorm) when squaredNorm > 0)."""
    x, y, z = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    z2 = (x * x + y * y) + z * z
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(z2 > 0, z / np.sqrt(z2), z).astype(F)


# ------------------------------------------------------------------ RANSAC
def plane_dist(c: np.ndarray, pts: np.ndarray) -> np.ndarray:
    """Eigen's SSE dot of c [..., 4] with (x, y, z, 1): (c0 x + c2 z) + (c1 y + c3)."""
    c = c.astype(F)
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    return (c[..., 0:1] * x + c[..., 2:3] * z) + (c[..., 1:2] * y + c[..., 3:4] * F(1))


def sample_good(p0, p1, p2) -> bool:
    with np.errstate(invalid="ignore", divide="ignore"):
        d = (p1[:3] - p0[:3]) / (p2[:3] - p0[:3])
    return bool(d[0] != d[1] or d[2] != d[1])


def model_coefficients(p0, p1, p2) -> np.ndarray:
    a = (p1[:3] - p0[:3]).astype(F); b = (p2[:3] - p0[:3]).astype(F)
    c = np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0], 0], F)
    z = (c[0] * c[0] + c[2] * c[2]) + (c[1] * c[1] + c[3] * c[3])
    if z > 0:
        c = (c / np.sqrt(z)).astype(F)
    c[3] = F(-1) * ((c[0] * p0[0] + c[2] * p0[2]) + (c[1] * p0[1] + c[3] * F(1)))
    return c


def stop_rule(counts, flags, n_points: int, probability: float = 0.99, max_iterations: int = 10000) -> dict:
    """computeModel's loop on hypotheses given in draw order."""
    it, skipped, best_count, best, k = 0, 0, -(2 ** 31 - 1), -1, 1.0
    log_p = math.log(1.0 - probability)
    one_over = 1.0 / float(n_points)
    max_skip = max_iterations * 10
    eps = np.finfo(np.float64).eps
    consumed = 0
    for c, f in zip(counts, flags):
        if not (it < k and skipped < max_skip):   # the while condition, before every draw
            break
        consumed += 1
        if f < 0:
            return dict(consumed=consumed, best=best, iterations=it, skipped=skipped, best_count=best_count)
        if f == 0:
            skipped += 1
            continue
        if c > best_count:
            best_count, best = int(c), consumed - 1
            w = float(c) * one_over
            p_no = 1.0 - math.pow(w, 3.0)
            p_no = min(1.0 - eps, max(eps, p_no))
            k = log_p / math.log(p_no)
        it += 1
        if it > max_iterations:
            return dict(consumed=consumed, best=best, iterations=it, skipped=skipped, best_count=best_count)
    ended = not (it < k and skipped < max_skip)
    return dict(consumed=consumed if ended else -1, best=best, iterations=it, skipped=skipped, best_count=best_count)


def ransac(pts: np.ndarray, threshold: float, probability: float = 0.99, max_iterations: int = 10000, chunk: int = 256):
    """RandomSampleConsensus<SampleConsensusModelPlane>::computeModel + getInliers.  Hypotheses are drawn and counted in
    chunks; the stop rule decides how many are used."""
    n = pts.shape[0]
    rng = MT19937(12345)
    shuf = np.arange(n, dtype=np.int64)
    idx, flags, coeffs, counts = [], [], [], []
    done = False
    while True:
        new_c = []
        for _ in range(chunk):
            if done:
                break
            good = False
            for _t in range(1000):
                for i in range(3):
                    j = i + (rng.next() >> 1) % (n - i)
                    shuf[i], shuf[j] = shuf[j], shuf[i]
                s = shuf[:3].copy()
                if sample_good(pts[s[0]], pts[s[1]], pts[s[2]]):
                    good = True
                    break
            if not good:
                idx.append([-1, -1, -1]); flags.append(-1); new_c.append(np.zeros(4, F)); done = True
                break
            idx.append(list(s))
            p0, p1, p2 = pts[s[0]], pts[s[1]], pts[s[2]]
            if not sample_good(p0, p1, p2):
                flags.append(0); new_c.append(np.zeros(4, F))
            else:
                flags.append(1); new_c.append(model_coefficients(p0, p1, p2))
        if new_c:
            cc = np.stack(new_c)
            with np.errstate(invalid="ignore"):
                cnt = (np.abs(plane_dist(cc, pts)).astype(np.float64) < threshold).sum(axis=1)
            cnt = np.where(np.array(flags[-len(new_c):]) == 1, cnt, 0)
            coeffs.extend(cc); counts.extend(int(c) for c in cnt)
        st = stop_rule(counts, flags, n, probability, max_iterations)
        if st["consumed"] >= 0 or done:
            break
    m = st["consumed"] if st["consumed"] >= 0 else len(flags)
    out = dict(idx=np.array(idx[:m], np.int64).reshape(-1, 3), flags=np.array(flags[:m], np.int32),
               counts=np.array(counts[:m], np.int64), iterations=st["iterations"], skipped=st["skipped"], best=st["best"])
    if st["best"] < 0:
        out.update(coeffs=None, inliers=np.zeros(0, np.int64))
        return out
    c = coeffs[st["best"]]
    with np.errstate(invalid="ignore"):
        inl = np.nonzero(np.abs(plane_dist(c[None, :], pts)[0]).astype(np.float64) < threshold)[0]
    out.update(coeffs=c.astype(F), inliers=inl)
    return out


# ------------------------------------------------------------------ scenes
def rot_x(deg: float) -> np.ndarray:
    a = math.radians(deg)
    return np.array([[1, 0, 0], [0, math.cos(a), -math.sin(a)], [0, math.sin(a), math.cos(a)]])


def scene(seed: int, n_ground: int = 20000, ground_z: float = -1.8, roll_deg: float = 0.0, radius: float = 25.0,
          walls: int = 0, platform: int = 0, noise: float = 0.01) -> np.ndarray:
    """A level ground disc at ground_z (sensor frame), optional vertical walls and a raised 10 x 10 m platform 0.5 m above the
    ground with `platform` points, the whole cloud rolled by roll_deg about x.  [n,4] float32, intensity in [0, 1)."""
    rng = np.random.default_rng(seed)
    parts = []
    r = radius * np.sqrt(rng.random(n_ground)); th = 2 * np.pi * rng.random(n_ground)
    parts.append(np.stack([r * np.cos(th), r * np.sin(th), ground_z + noise * rng.standard_normal(n_ground)], 1))
    if platform:
        parts.append(np.stack([rng.uniform(3, 13, platform), rng.uniform(-5, 5, platform),
                               ground_z + 0.5 + noise * rng.standard_normal(platform)], 1))
    for w in range(walls):
        m = 3000
        a = rng.uniform(0, 2 * np.pi); d = rng.uniform(5, 20)
        t = rng.uniform(-8, 8, m)
        c, s = math.cos(a), math.sin(a)
        parts.append(np.stack([d * c - t * s, d * s + t * c, rng.uniform(ground_z, ground_z + 4, m)], 1))
    xyz = np.concatenate(parts) @ rot_x(roll_deg).T
    xyz = xyz[rng.permutation(xyz.shape[0])]
    return np.concatenate([xyz, rng.random((xyz.shape[0], 1))], 1).astype(F)


# ------------------------------------------------------------------ the whole detector
def detect(pts: np.ndarray, p: dict) -> dict:
    pts = np.ascontiguousarray(pts, F)
    r = dict(found=False, reason=EMPTY, coeffs=None, prefiltered=pts[:0], clip_idx=np.zeros(0, np.int64),
             cand_idx=np.zeros(0, np.int64), clipped=pts[:0], candidates=pts[:0], inliers=pts[:0], ransac=None)
    if pts.shape[0] == 0:
        return r
    pre = prefilter(pts, p) if p["prefilter_leaf"] > 0 else pts
    r["prefiltered"] = pre
    ci = np.nonzero(clip_mask(pre, p))[0]
    clipped = pre[ci]
    r["clip_idx"], r["clipped"] = ci, clipped
    if p["use_normal_filtering"]:
        nrm, cov6, nbr = normals(clipped[:, :3], p["viewpoint_z"])
        r["normals"], r["cov6"], r["nbr"] = nrm, cov6, nbr
        nz = normal_nz(nrm)
        r["abs_nz"] = np.abs(nz)
        with np.errstate(invalid="ignore"):
            keep = np.abs(nz).astype(np.float64) > math.cos(p["normal_filter_deg"] * math.pi / 180.0)
        cand_idx = np.nonzero(keep)[0]
    else:
        cand_idx = np.arange(clipped.shape[0])
    cand = clipped[cand_idx]
    r["cand_idx"], r["candidates"] = cand_idx, cand
    if cand.shape[0] < p["floor_pts_thresh"]:
        r["reason"] = FEW_CANDIDATES
        return r
    if cand.shape[0] < 3:
        r["reason"] = NO_MODEL
        return r
    rs = ransac(cand, p["ransac_threshold"], p["ransac_probability"], p["ransac_max_iterations"])
    r["ransac"] = rs
    if rs["coeffs"] is None:
        r["reason"] = NO_MODEL
        return r
    c = rs["coeffs"].copy()
    r["coeffs"] = c
    r["inliers"] = cand[rs["inliers"]]
    if rs["inliers"].size < p["floor_pts_thresh"]:
        r["reason"] = FEW_INLIERS
        return r
    if float(abs(c[2])) < math.cos(p["floor_normal_deg"] * math.pi / 180.0):
        r["reason"] = NOT_VERTICAL
        return r
    if c[2] < 0:
        r["coeffs"] = (c * F(-1)).astype(F)
    r["found"], r["reason"] = True, FOUND
    return r
