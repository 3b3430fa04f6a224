"""CPU: the voxelizer oracle (oracle/vfe.py, OracleVoxelizer) against a brute-force restatement, on the edge sets of
tests/vfe_edges.py that the GPU tests hold the device to.

The restatement keeps the window as a list of frames (newest first) and transforms it point by point in exact rational
arithmetic, each fp32 operation rounded to nearest even from the exact value; it voxelizes by walking the points in order
into a dict keyed by cell, whose insertion order is the voxel order.  The oracle must give the same totals, the same
window bits, and the same voxel rows, counts and fp16 feature bits (any NaN equal to any NaN)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import vfe_edges as E
from oracle.vfe import FAR_ROW_XYZ, OracleVoxelizer, fma32

F32 = np.float32


def _round32(q: Fraction) -> np.float32:
    """q rounded to the nearest fp32, ties to even (q within the finite fp32 range)."""
    d = F32(float(q))                                    # at most one fp32 step away from the answer
    cands = [np.nextafter(d, F32(-np.inf)), d, np.nextafter(d, F32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c, F32).view(np.uint32)) & 1))


def _exact(*v):
    return all(math.isfinite(float(x)) for x in v)


def _mul(a, b):
    if _exact(a, b):
        return _round32(Fraction(float(a)) * Fraction(float(b)))
    with np.errstate(invalid="ignore"):                  # 0 * inf
        return F32(np.float64(a) * np.float64(b))


def _add(a, b):
    if _exact(a, b):
        return _round32(Fraction(float(a)) + Fraction(float(b)))
    with np.errstate(invalid="ignore"):                  # inf - inf
        return F32(np.float64(a) + np.float64(b))


def _fma(a, b, c):
    if _exact(a, b, c):
        return _round32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))
    with np.errstate(invalid="ignore"):
        return F32(np.float64(a) * np.float64(b) + np.float64(c))


class Restated:
    """The sliding window as frames: a realtime frame drops the oldest frame, gets max(min(n, max_points - rows left), 1)
    rows (the far row when it brings none), and the frames it joins are moved by the motion, time + 0.1."""

    def __init__(self, max_points, frames, nf):
        self.M, self.F, self.nf = max_points, frames, nf
        self.frames = [np.zeros((0, nf), F32)] * frames

    def accumulate(self, pts, m, realtime=True):
        pts = np.asarray(pts, F32).reshape(-1, self.nf)
        if not realtime:
            self.frames = [pts[:self.M].copy()] + [np.zeros((0, self.nf), F32)] * (self.F - 1)
            return self.total()
        keep = self.frames[:self.F - 1]
        left = sum(f.shape[0] for f in keep)
        n = max(min(pts.shape[0], self.M - left), 1)
        if pts.shape[0] == 0:
            pts = np.zeros((1, self.nf), F32)
            pts[0, :3] = FAR_ROW_XYZ
        m = np.asarray(m, F32).ravel()
        moved = []
        for fr in keep:
            out = fr.copy()
            for i, p in enumerate(fr):
                for r in range(3):
                    t = _mul(m[4 * r + 1], p[1])
                    t = _fma(m[4 * r], p[0], t)
                    t = _fma(m[4 * r + 2], p[2], t)
                    out[i, r] = _add(t, m[4 * r + 3])
                if self.nf > 4:
                    out[i, 4] = F32(float(p[4]) + 0.1)
            moved.append(out)
        self.frames = [pts[:n].copy()] + moved
        return self.total()

    def total(self):
        return sum(f.shape[0] for f in self.frames)

    def window(self):
        return np.concatenate(self.frames, 0)


def restated_voxels(o: OracleVoxelizer, win, zyx=True):
    """Point by point: the range test (NaN passes), the cell floor((p - min) / vs) in fp32 (NaN -> 0), the grid test; then
    the first max_ppv points of each cell summed in point order in fp32, divided by their count, rounded to fp16."""
    cells = {}
    for i, p in enumerate(win):
        c, ok = [], True
        for a in range(3):
            v = p[a]
            if v < o.mn[a] or v >= o.mx[a]:
                ok = False
                break
            with np.errstate(invalid="ignore", over="ignore"):
                q = np.floor((v - o.mn[a]) / o.vs[a])
            k = 0 if math.isnan(q) else int(q) if math.isfinite(q) else -1
            if not 0 <= k < o.gs[a]:
                ok = False
                break
            c.append(k)
        if ok:
            cells.setdefault(tuple(c), []).append(i)
    rows = list(cells.items())[:o.max_voxels]
    feat = np.zeros((len(rows), o.nf), np.float16)
    idx = np.zeros((len(rows), 4), np.uint32)
    npts = np.zeros(len(rows), np.uint32)
    for v, (c, members) in enumerate(rows):
        use = members[:o.max_ppv]
        with np.errstate(invalid="ignore", over="ignore"):
            acc = win[use[0]].copy()
            for j in use[1:]:
                acc = acc + win[j]
            feat[v] = (acc / F32(len(use))).astype(np.float16)
        idx[v, 1:] = c[::-1] if zyx else c
        npts[v] = len(use)
    return feat, idx, npts


def _same_bits(a, b):
    u = np.uint16 if a.dtype == np.float16 else np.uint32
    return ((a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))).all()


def _check_voxels(o, win, zyx=True):
    of, oi, on = o.voxelize(points=win, zyx=zyx)
    rf, ri, rn = restated_voxels(o, win, zyx)
    np.testing.assert_array_equal(oi, ri)
    np.testing.assert_array_equal(on, rn)
    assert of.shape == rf.shape and _same_bits(of, rf)
    return of, oi, on


def test_fma32_is_correctly_rounded():
    """Random operands, and operands built so that the float64 sum lands exactly halfway between two floats while the
    exact value does not (where rounding the float64 sum again would be wrong)."""
    rng = np.random.default_rng(0)
    a = rng.uniform(-2, 2, 3000).astype(F32); b = rng.uniform(-2, 2, 3000).astype(F32); c = rng.uniform(-2, 2, 3000).astype(F32)
    # c = 1 + odd * 2^-23 and a*b = 2^-24 - 2^-60: the exact sum lies just under the midpoint c + 2^-24 and rounds to c,
    # but its float64 rounding is the midpoint itself, which ties to the even neighbour c + 2^-23
    a2 = np.full(64, F32(1.0 + 2.0 ** -18))
    b2 = np.full(64, F32(2.0 ** -24 * (1.0 - 2.0 ** -18)))
    c2 = (1.0 + (2 * np.arange(64) + 1) * 2.0 ** -23).astype(F32)
    with np.errstate(over="ignore"):
        naive = (a2.astype(np.float64) * b2.astype(np.float64) + c2.astype(np.float64)).astype(F32)
    for x, y, z in ((a, b, c), (a2, b2, c2), (-a2, b2, -c2)):
        got = fma32(x, y, z)
        want = np.array([_fma(p, q, r) for p, q, r in zip(x, y, z)], F32)
        assert _same_bits(got, want)
    assert (naive != c2).all() and _same_bits(fma32(a2, b2, c2), c2)


@pytest.mark.parametrize("max_points", [40, 100])
@pytest.mark.parametrize("frames", [1, 2, 3, 4])
def test_window_totals_and_voxels_at_the_cap(max_points, frames):
    rng = np.random.default_rng(max_points + frames)
    M = max_points
    o, r = OracleVoxelizer(max_points=M, max_frames=frames, max_voxels=100000), Restated(M, frames, 5)
    peak = 0
    for step, n in enumerate([M, M, M, M, 0, M // 2, 3 * M, 0, 0, 1, M - 1, M, 2, 0, M, M]):
        pts = E.cloud(rng, n, 5)
        mot = E.motion(rng)
        t = o.accumulate(pts, mot)
        assert t == r.accumulate(pts, mot) and 1 <= t <= M + frames - 1
        peak = max(peak, t)
        assert _same_bits(o.buf[:t], r.window())
        _check_voxels(o, o.buf[:t], zyx=bool(step % 2))
    assert peak == M + frames - 1
    for n in (M + 7, 0):
        pts = E.cloud(rng, n, 5)
        assert o.accumulate(pts, None, realtime=False) == r.accumulate(pts, None, realtime=False) == min(n, M)
        mot = E.motion(rng)
        pts = E.cloud(rng, 3, 5)
        assert o.accumulate(pts, mot) == r.accumulate(pts, mot)
        assert _same_bits(o.buf[:o.total], r.window())


@pytest.mark.parametrize("nf", [4, 5, 8])
def test_nonfinite_points(nf):
    rng = np.random.default_rng(11 + nf)
    o, r = OracleVoxelizer(nf=nf, max_frames=3), Restated(500000, 3, nf)
    for f, full in enumerate(E.nonfinite_frames(rng, nf)):
        bad = ~np.isfinite(full).all(1)
        pts = np.concatenate([full[~bad][:300], full[bad]])              # every non-finite row, some finite ones
        mot = E.motion(rng, yaw_only=f == 1)
        assert o.accumulate(pts, mot) == r.accumulate(pts, mot)
        win = o.buf[:o.total]
        assert _same_bits(win, r.window())
        feat, idx, npts = _check_voxels(o, win)
        nan = np.isnan(feat[:, :3].astype(F32)).any(1)
        assert nan.any() and (idx[nan][:, 1:] == 0).any(1).all()


@pytest.mark.parametrize("grid", list(E.GRIDS))
def test_faces(grid):
    gp = E.GRIDS[grid]
    o = OracleVoxelizer(min_range=gp["min_range"], max_range=gp["max_range"], voxel_size=gp["voxel_size"])
    pts = E.face_points(gp)
    o.accumulate(pts, None, realtime=False)
    feat, idx, npts = _check_voxels(o, o.buf[:o.total])
    mn = np.asarray(gp["min_range"], F32)
    on_min = (pts[:, :3] == mn).any(1) & ((pts[:, :3] < np.asarray(gp["max_range"], F32)).all(1))
    assert 0 < feat.shape[0] < pts.shape[0] and on_min.any()


@pytest.mark.parametrize("nf", [4, 5, 8])
@pytest.mark.parametrize("ppv", [1, 3, 5])
def test_shapes(nf, ppv):
    rng = np.random.default_rng(nf * 10 + ppv)
    o = OracleVoxelizer(nf=nf, max_ppv=ppv, max_frames=2)
    r = Restated(500000, 2, nf)
    for f in range(2):
        pts = E.cloud(rng, 600, nf)
        mot = E.motion(rng)
        assert o.accumulate(pts, mot) == r.accumulate(pts, mot)
        assert _same_bits(o.buf[:o.total], r.window())
        for zyx in (True, False):
            feat, idx, npts = _check_voxels(o, o.buf[:o.total], zyx)
        assert npts.max() == ppv


def test_fp16_features():
    v = E.fp16_values(np.random.default_rng(5))
    n = v.shape[0]
    pts = np.zeros((2 * n, 5), F32)
    pts[:, 0] = np.repeat(F32(-59.95) + F32(0.1) * np.arange(n, dtype=F32), 2)
    pts[::2, 1] = 10.05                                                    # x cell j: a first point
    pts[1::2, 1] = 10.05 + 3 * (np.arange(n) % 2 == 0)                     # and a second one, in its voxel for odd j
    pts[:, 3] = np.concatenate([v, v[::-1]]).reshape(2, n).T.ravel()
    pts[:, 4] = np.roll(pts[:, 3], 3)
    o = OracleVoxelizer()
    o.accumulate(pts, None, realtime=False)
    feat, idx, npts = _check_voxels(o, o.buf[:o.total])
    assert (npts == 1).any() and (npts == 2).any()
