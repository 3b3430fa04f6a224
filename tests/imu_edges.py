"""TEST INFRASTRUCTURE: the IMU stage (ImuProcess, row N1) driven side by side through the product (lsdreg.ImuProcess), the
COMPILED reference class (oracle/_ref/libref_ikfom.so, IMU_Processing.hpp:167-450 unmodified) and the numpy restatement
(oracle/imu.py), on streams built to reach the edges of the segment walk of UndistortPcl:

* the repeated compensation of the earliest point (`if (it_pcl == begin) break;`, IMU_Processing.hpp:403, which leaves
  the iterator on that point for every remaining segment) with chains of 3 to 12 compensations;
* point times equal to an IMU pose offset (the strict `curvature / 1000 > head->offset_time`), and one float ulp either
  side;
* IMU samples stamped after lidar_end_time (`note = -1`, a pose list that is not monotone at its tail) and points timed
  after the scan end;
* the forward propagation's stale samples, `head.stamp < last_lidar_end_time` dt, the prediction across a gap to the scan
  start and the `min(1.0, dt)` clamp; IMU_init's "not stable, reset" path and the INS velocity seed;
* the device's own limits: kMaxImuPoses = 256 IMU poses per scan, the earliest-point key (times <= 0, -0.0, ties), point
  counts that are not a multiple of the block size, n = 0 and 1.

Points carry their input index in the intensity channel (exact below 2^24; every side passes intensity through), so the
reference's time-sorted cloud maps back to input order and every point is compared with its own counterpart.

Bars (those of tests/test_oracle_ikfom.py, where the restatement meets the same reference): state 1e-11, P rtol 1e-9 /
atol 1e-14, the IMU pose list as there; points per input index within 2 float32 ulp of the coordinate's magnitude, 2 k ulp
for the point compensated k times.

Ties.  When several points share the earliest time and that time is past the first IMU pose, the reference compensates
repeatedly whichever of them std::sort put first (libstdc++'s introsort: unspecified among equal keys); the product
compensates the lowest input index (the restatement's stable sort does the same).  What is checked there: exactly one
point of the tied group carries the chain on each side, every other point matches per index, and the product's chained
point equals the restatement's.

Used by tests/test_gpu_imu_edges.py (H100 sizes) and tests/simt/fuzz_imu.py (the same cases at emulator sizes)."""
import math

import numpy as np

import lsdreg
from lsdreg import synth
from oracle import eskf as E
from oracle import oracle as O
from oracle.imu import OracleImuProcess, exp_rodrigues

R = O.ref_ikfom
EXT_R = synth.rot_from_rpy(0.02, -0.01, 0.05)
EXT_T = np.array([0.3, -0.1, 0.2])
OMEGA = np.array([0.05, -0.03, 1.0])          # rad/s once moving: about 1 rad/s of yaw, a little roll and pitch
ACCEL = np.array([0.8, 0.3, 0.0])             # m/s^2 once moving
MAX_POSES = 256                               # kMaxImuPoses, csrc/imu.cu


class RefImu:
    """The compiled ImuProcess + esekf (oracle/ref_ikfom.cpp)."""

    def __init__(self, ext_R, ext_t, undistort=True):
        self.h = R.ref_imu_create(np.ascontiguousarray(ext_R, np.float64).reshape(9), np.ascontiguousarray(ext_t, np.float64), 0.1, 0.1, 1e-4, 1e-4,
                                  int(undistort))

    def __del__(self):
        if getattr(self, "h", None):
            R.ref_imu_destroy(self.h); self.h = None

    def process(self, m, x26, P):
        pts = np.ascontiguousarray(m["points"], np.float32); tms = np.ascontiguousarray(m["time_ms"], np.float32)
        out = np.zeros_like(pts); out_t = np.zeros_like(tms)
        imu = np.ascontiguousarray(m["imu"], np.float64).reshape(-1, 7)
        iv = None if m.get("ins_vel") is None else np.ascontiguousarray(m["ins_vel"], np.float64)
        n = R.ref_imu_process(self.h, imu, imu.shape[0], None if iv is None else iv.ctypes.data, float(m["lidar_beg_time"]), float(m["lidar_end_time"]),
                              pts, tms, pts.shape[0], x26, P, out, out_t)
        return out[:n], out_t[:n]

    def poses(self):
        buf = np.zeros((4096, 22))
        n = R.ref_imu_get_poses(self.h, buf, 4096)
        return buf[:n]


# ---------------------------------------------------------------- streams
def imu_rows(rng, stamps, moving, omega=OMEGA):
    """IMU samples: gyr rad/s, acc in g-units (+1 g on z at rest)."""
    imu = np.zeros((len(stamps), 7))
    imu[:, 0] = stamps
    imu[:, 1:4] = rng.normal(0, 0.002, (len(stamps), 3)) + (omega if moving else 0.0)
    imu[:, 4:7] = np.array([0.0, 0.0, 1.0]) + rng.normal(0, 0.002, (len(stamps), 3)) + (ACCEL / 9.81 if moving else 0.0)
    return imu


def cloud(rng, n):
    """n points up to ~50 m away; intensity = input index."""
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = rng.uniform(-50, 50, (n, 3)); pts[:, 2] *= 0.2
    pts[:, 3] = np.arange(n, dtype=np.float32)
    return pts


def uniform_times(lo, hi):
    """Times uniform in (lo, hi) ms with exactly one point at lo (a unique earliest point)."""
    def f(rng, n, k):
        t = rng.uniform(lo, hi, n).astype(np.float32)
        t[t <= np.float32(lo)] = np.float32(hi)
        if n:
            t[rng.integers(0, n)] = np.float32(lo)
        return t
    return f


def stream(rng, n_pts, times, n_moving=4, hz=200, period=0.1, t0=0.0, off=0.0, imu_lead=0.0, n_init=None, n_pts_init=8):
    """Packages of a platform that stands still until the IMU is initialised (> 100 samples) and then moves.  Scans abut
    ([t0 + f period, t0 + (f + 1) period]); the IMU runs on a grid off + j / hz; a package carries the samples in
    (previous end + imu_lead, end + imu_lead].  times(rng, n, k) gives the point times of moving scan k."""
    per = int(round(hz * period))
    if n_init is None:
        n_init = (100 + per - 1) // per + 1                 # one still scan is undistorted too
    out, j = [], int(math.floor((t0 + imu_lead - off) * hz + 1e-6)) + 1
    for f in range(n_init + n_moving):
        beg, end = t0 + f * period, t0 + (f + 1) * period
        j1 = int(math.floor((end + imu_lead - off) * hz + 1e-6))
        stamps = off + np.arange(j, j1 + 1) / hz
        j = j1 + 1
        moving = f >= n_init
        n = n_pts if moving else n_pts_init
        tms = times(rng, n, f - n_init) if moving else rng.uniform(0, period * 1000, n).astype(np.float32)
        out.append(dict(lidar_beg_time=beg, lidar_end_time=end, points=cloud(rng, n), time_ms=tms, imu=imu_rows(rng, stamps, moving), ins_vel=None))
    return out


# ---------------------------------------------------------------- one compensation, restated for the tie / chain checks
def compensate(p, t, poses, x_end, heads):
    """IMU_Processing.hpp:386-401 for the segments with the given heads, in that order, rounding to float32 after each."""
    Rend = E.quat_to_R(x_end[3:7]); RL = E.quat_to_R(x_end[7:11]); tL = x_end[11:14]; pend = x_end[0:3]
    q = np.asarray(p[:3], np.float32)
    for h in heads:
        hd, tl = poses[h], poses[h + 1]
        dt = t - hd[0]
        Ri = hd[13:22].reshape(3, 3) @ exp_rodrigues(tl[4:7], dt)
        Tei = hd[10:13] + hd[7:10] * dt + 0.5 * tl[1:4] * dt * dt - pend
        q = (RL.T @ (Rend.T @ (Ri @ (RL @ q.astype(np.float64) + tL) + Tei) - tL)).astype(np.float32)
    return q


def heads_below(t, poses):
    """Segment heads (descending) whose offset time is below t: the first is the point's own segment, all of them are
    the earliest point's chain."""
    return [h for h in range(len(poses) - 2, -1, -1) if t > poses[h, 0]]


def ulp_ok(a, b, k):
    """|a - b| <= 2 max(k, 1) float32 ulp of the coordinate's magnitude, per coordinate."""
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    mag = np.maximum(np.abs(a), np.abs(b)).astype(np.float32)
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) <= 2 * max(k, 1) * np.spacing(mag).astype(np.float64)


def _assert_ulp(what, a, b, k, idx):
    """Points a and b (rows = the input indices idx) within 2 max(k, 1) float32 ulp per coordinate."""
    d = np.abs(a[:, :3].astype(np.float64) - b[:, :3])
    mag = np.maximum(np.abs(a[:, :3]), np.abs(b[:, :3])).astype(np.float32)
    bar = 2 * np.maximum(k, 1)[:, None] * np.spacing(mag).astype(np.float64)
    bad = np.flatnonzero((d > bar).any(axis=1))
    assert bad.size == 0, (what, idx[bad[:5]], a[bad[:5]], b[bad[:5]], k[bad[:5]])


def by_index(sorted_cloud, n):
    """A time-sorted cloud back in input order through the index in the intensity channel."""
    idx = sorted_cloud[:, 3].astype(np.int64)
    assert np.array_equal(np.sort(idx), np.arange(n)), "intensity (input index) not carried through"
    out = np.empty_like(sorted_cloud)
    out[idx] = sorted_cloud
    return out, idx


# ---------------------------------------------------------------- the three implementations in lock step
class Trio:
    def __init__(self, ext_R=EXT_R, ext_t=EXT_T, undistort=True, oracle_subset=None):
        self.g = lsdreg.ImuProcess(ext_R=ext_R, ext_t=ext_t, undistort=int(undistort))
        self.r = RefImu(ext_R, ext_t, undistort)
        self.o = OracleImuProcess(ext_R=ext_R, ext_t=ext_t, undistort=undistort)
        self.undistort = undistort
        self.xo, self.Po = E.State(), E.init_P()
        self.xr, self.Pr = self.xo.to_vec().copy(), self.Po.copy()
        self.xg, self.Pg = self.xr.copy(), self.Pr.copy()
        self.oracle_subset = oracle_subset      # above this many points the restatement sees every 97th point (+ the earliest)
        self.n_und = 0
        self.chains = []                        # per undistorted scan: (earliest time's chain length, |chain - one compensation| in m)

    def step(self, m, points=None, time_ms=None):
        """One package through all three; asserts state, P, pose list and every point.  points / time_ms override what
        the product is handed (CUDA tensors for the device path).  -> True if the scan was undistorted, None while the
        IMU initialises (or the package has no IMU sample)."""
        n = len(m["points"])
        out_r, t_r = self.r.process(m, self.xr, self.Pr)
        mo = m
        sub = None
        if self.oracle_subset is not None and n > self.oracle_subset:
            sub = np.unique(np.concatenate([np.arange(0, n, 97), [int(np.argmin(m["time_ms"]))]]))
            mo = dict(m, points=m["points"][sub], time_ms=m["time_ms"][sub])
        out_o = self.o.process(mo, self.xo, self.Po)
        st, self.xg, self.Pg, n_g = self.g.process(m["imu"], m["lidar_beg_time"], m["lidar_end_time"], m["points"] if points is None else points,
                                                   m["time_ms"] if time_ms is None else time_ms, self.xg, self.Pg, ins_vel=m.get("ins_vel"))
        for x, P in ((self.xg, self.Pg), (self.xo.to_vec(), self.Po)):
            np.testing.assert_allclose(x, self.xr, rtol=0, atol=1e-11)
            np.testing.assert_allclose(P, self.Pr, rtol=1e-9, atol=1e-14)
        if out_o is None:
            assert st == lsdreg.IMU_INITIALIZING and n_g == 0 and len(out_r) == 0, (st, n_g, len(out_r))
            return None
        assert st == lsdreg.OK and n_g == n and len(out_r) == n, (st, n_g, len(out_r), n)
        pr, pg = self.r.poses(), self.g.poses()
        po = np.array([np.concatenate([[q["t"]], q["acc"], q["gyr"], q["vel"], q["pos"], q["rot"].reshape(9)]) for q in self.o.IMUpose])
        assert len(pr) == len(pg) == len(po), (len(pr), len(pg), len(po))
        for side in (pg, po):
            np.testing.assert_allclose(side[:, 0], pr[:, 0], rtol=0, atol=1e-12)
            # the reference never initialises acc_s_last: IMUpose[0].acc of the first scan is garbage (and unused, :379)
            a0 = 1 if self.n_und == 0 else 0
            np.testing.assert_allclose(side[a0:, 1:4], pr[a0:, 1:4], rtol=0, atol=1e-10)
            np.testing.assert_allclose(side[:, 4:7], pr[:, 4:7], rtol=0, atol=1e-12)
            np.testing.assert_allclose(side[:, 7:13], pr[:, 7:13], rtol=0, atol=1e-11)
            np.testing.assert_allclose(side[:, 13:22], pr[:, 13:22], rtol=0, atol=1e-12)
        self.n_und += 1
        cg = self.g.cloud()
        assert cg.shape == (n, 4)
        np.testing.assert_array_equal(cg[:, 3], m["points"][:, 3])
        if n == 0:
            return True
        ref, ridx = by_index(out_r, n)
        np.testing.assert_array_equal(np.sort(m["time_ms"]), t_r)
        np.testing.assert_array_equal(ref[:, 3], m["points"][:, 3])
        seen, oo = self._oracle_by_index(out_o, sub, n)
        if not self.undistort:
            np.testing.assert_array_equal(cg, m["points"])               # input order, untouched
            np.testing.assert_array_equal(ref, m["points"])
            np.testing.assert_array_equal(oo, m["points"][seen])
            return True
        self._check_points(m, pr, ref, ridx, cg, (seen, oo))
        return True

    @staticmethod
    def _oracle_by_index(out_o, sub, n):
        """The restatement's sorted cloud in input order: (the input indices it saw, its points in that order)."""
        if sub is None:
            return np.arange(n), by_index(out_o, n)[0]
        o = np.empty_like(out_o)
        o[np.searchsorted(sub, out_o[:, 3].astype(np.int64))] = out_o
        return sub, o

    def _check_points(self, m, pr, ref, ridx, cg, oracle):
        n = len(m["points"])
        tms = m["time_ms"].astype(np.float32)
        t = tms.astype(np.float64) / 1000.0
        k = (t[:, None] > pr[None, :-1, 0]).any(axis=1).astype(np.int64)   # compensated once, or not at all
        tmin = tms.min()
        group = np.flatnonzero(tms == tmin)
        chain = heads_below(float(tmin) / 1000.0, pr)
        first_ref = int(ridx[0])                                         # whom the reference's sort put first
        assert first_ref in set(group.tolist())
        k[first_ref] = max(len(chain), 1)
        tied_chain = len(group) > 1 and len(chain) > 1
        if len(chain) > 1:
            g0 = int(group[0])
            one = compensate(m["points"][g0], float(t[g0]), pr, self.xr, chain[:1])
            full = compensate(m["points"][g0], float(t[g0]), pr, self.xr, chain)
            self.chains.append((len(chain), float(np.abs(full.astype(np.float64) - one).max())))
        else:
            self.chains.append((len(chain), 0.0))
        plain = np.ones(n, bool)
        if tied_chain:
            plain[group] = False
            one = {int(g): compensate(m["points"][g], float(t[g]), pr, self.xr, chain[:1]) for g in group}
            full = {int(g): compensate(m["points"][g], float(t[g]), pr, self.xr, chain) for g in group}
            for side, name, want in ((ref, "reference", first_ref), (cg, "product", int(group[0]))):
                carriers = []
                for g in one:
                    is_full, is_one = ulp_ok(side[g, :3], full[g], len(chain)).all(), ulp_ok(side[g, :3], one[g], 1).all()
                    assert is_full != is_one, (name, g, side[g], one[g], full[g])
                    carriers += [g] if is_full else []
                assert carriers == [want], (name, carriers, want)   # the product: the lowest index of the tied group
            for g in one:
                if g not in (first_ref, int(group[0])):
                    assert ulp_ok(cg[g, :3], ref[g, :3], 1).all(), (g, cg[g], ref[g])
        # every other point per input index
        idx = np.flatnonzero(plain)
        _assert_ulp("product vs reference", cg[idx], ref[idx], k[idx], idx)
        # the restatement: against the reference on every point it saw, and equal to the product everywhere (its stable
        # sort puts the lowest index of a tied group first, like the product)
        sub, oo = oracle
        keep = plain[sub]
        _assert_ulp("restatement vs reference", oo[keep], ref[sub][keep], k[sub][keep], sub[keep])
        _assert_ulp("product vs restatement", cg[sub], oo, np.where(np.isin(sub, group), max(len(chain), 1), k[sub]), sub)

    def run(self, pkgs):
        return [self.step(m) for m in pkgs]


# ---------------------------------------------------------------- the cases
def case_leading_gap(big, gap_ms):
    """No point earlier than gap_ms: the earliest point is compensated by its own segment and again by every segment
    below it (3 times at 12.5 ms, 12 at 57.5 ms on a 200 Hz IMU)."""
    rng = np.random.default_rng(11)
    tr = Trio()
    tr.run(stream(rng, 6000 if big else 700, uniform_times(gap_ms, 100.0)))
    moving = tr.chains[-4:]
    want = int(math.ceil(gap_ms / 5.0))
    assert all(c == want for c, _ in moving), moving
    assert all(d > 1e-3 for _, d in moving), moving          # the chain moves the point by more than a millimetre


def case_head_ties(big):
    """beg multiple of 1/8 s, 128 Hz IMU: pose offsets k / 128 s are exact, and so are point times k * 1000 / 128 ms
    (and their / 1000); points exactly on a pose offset and one float ulp either side."""
    def times(rng, n, k):
        grid = (np.arange(0, 17) * np.float32(1000.0 / 128.0)).astype(np.float32)
        on = grid[rng.integers(0, 17, n)]
        side = rng.integers(-1, 2, n)
        t = np.where(side < 0, np.nextafter(on, np.float32(-np.inf)), np.where(side > 0, np.nextafter(on, np.float32(np.inf)), on)).astype(np.float32)
        t[: n // 4] = rng.uniform(0, 125, n // 4).astype(np.float32)
        return t
    rng = np.random.default_rng(12)
    pkgs = stream(rng, 6000 if big else 700, times, hz=128, period=0.125, t0=0.125 * 40)
    for m in pkgs:
        assert np.all(np.asarray(m["imu"][:, 0]) * 128 == np.round(m["imu"][:, 0] * 128))
    tr = Trio()
    tr.run(pkgs)
    p = tr.r.poses()
    assert np.all(p[:, 0] * 128 == np.round(p[:, 0] * 128))   # exact offsets, so `t > offset` is decided on equality


def case_past_end(big):
    """The IMU is 2.5 ms ahead of the lidar: every package ends with a sample after lidar_end_time (note = -1, the last
    pose is earlier than the one before it); point times run to 130 ms on a 100 ms scan."""
    def times(rng, n, k):
        t = rng.uniform(0, 130, n).astype(np.float32)
        t[: n // 10] = rng.uniform(100, 130, n // 10).astype(np.float32)
        return t
    rng = np.random.default_rng(13)
    tr = Trio()
    pkgs = stream(rng, 6000 if big else 700, times, off=0.0025, imu_lead=0.0025)
    for m in pkgs:
        assert m["imu"][-1, 0] > m["lidar_end_time"]
    tr.run(pkgs)
    p = tr.r.poses()
    assert p[-1, 0] < p[-2, 0]


def case_stale_gaps(big):
    """Packages that repeat samples older than the last scan end; a 0.3 s and a 1.5 s lidar gap with the IMU running
    through it (the prediction to the scan start, then stale samples); a scan whose IMU has a 1.2 s hole (dt clamped
    to 1 s)."""
    rng = np.random.default_rng(14)
    n = 6000 if big else 700
    hz, off = 200, 0.001
    pkgs = stream(rng, n, uniform_times(0.5, 100.0), n_moving=2, off=off)
    last = pkgs[-1]
    t_end, j = last["lidar_end_time"], int(round((last["imu"][-1, 0] - off) * hz)) + 1

    def pkg(beg, end, stamps, times_lo=0.5, span=100.0):
        return dict(lidar_beg_time=beg, lidar_end_time=end, points=cloud(rng, n), time_ms=uniform_times(times_lo, span)(rng, n, 0),
                    imu=imu_rows(rng, stamps, True), ins_vel=None)

    def grid_to(end):
        nonlocal j
        j1 = int(math.floor((end - off) * hz + 1e-6))
        s = off + np.arange(j, j1 + 1) / hz
        j = j1 + 1
        return s

    extra = []
    for gap in (0.0, 0.3, 0.0, 1.5, 0.0):
        beg = t_end + gap
        end = beg + 0.1
        s = grid_to(end)
        if gap == 0.0 and extra:
            s = np.concatenate([extra[-1]["imu"][-4:, 0], s])           # repeated stale samples at the front
        extra.append(pkg(beg, end, s))
        t_end = end
    # the IMU stops for 1.2 s inside a 1.3 s scan: the segment across the hole is clamped to dt = 1
    beg = t_end; end = beg + 1.3
    s = grid_to(end)
    s = np.concatenate([s[:2], s[s > beg + 1.2]])
    extra.append(pkg(beg, end, s, span=1300.0))
    tr = Trio()
    tr.run(pkgs + extra)
    p = tr.r.poses()
    assert np.diff(p[:, 0]).max() > 1.0


def case_init_paths(big):
    """Motion during initialisation (mean gyro > 10 deg/s: "init is not stable, reset" and a fresh average), the INS
    velocity seed, and a scan whose package has no IMU sample (state, P and output count left alone; the next scan
    predicts across it)."""
    rng = np.random.default_rng(15)
    ins_vel = np.array([0.4, -0.2, 0.05])
    pkgs = stream(rng, 6000 if big else 700, uniform_times(7.5, 100.0), n_moving=5, n_init=8)
    for m in pkgs[:2]:
        m["imu"][:, 1:4] += np.array([0.0, 0.0, 0.5])                  # turning while the IMU initialises
    for m in pkgs:
        m["ins_vel"] = ins_vel
    pkgs[-2]["imu"] = np.zeros((0, 7))
    tr = Trio()
    res = []
    for m in pkgs:
        x0, P0 = tr.xg.copy(), tr.Pg.copy()
        res.append(tr.step(m))
        if res[-1] is None and len(res) <= 7:
            seeded = tr.xr[14:17].copy()
        if len(m["imu"]) == 0:
            assert res[-1] is None and np.array_equal(tr.xg, x0) and np.array_equal(tr.Pg, P0)
    first = next(i for i, r in enumerate(res) if r is not None)
    assert first == 7, first                                          # the two turning packages did not count
    np.testing.assert_array_equal(seeded, ins_vel)
    assert sum(r is not None for r in res) == 5


def case_times(big, kind):
    """Time-field edges: negative times, a single -0.0 among late points, every point at one time, ties inside the
    range, ties at the earliest time when that time is past the first IMU pose."""
    def times(rng, n, k):
        if kind == "negative":
            t = rng.uniform(-8, 100, n).astype(np.float32)
        elif kind == "negzero":
            t = uniform_times(12.5, 100.0)(rng, n, k)
            t[rng.integers(0, n)] = np.float32(-0.0)
        elif kind == "one_time":
            t = np.full(n, 37.5 + k, np.float32)
        elif kind == "mid_ties":
            t = uniform_times(0.25, 100.0)(rng, n, k)
            t[rng.integers(0, n, n // 3)] = np.float32([31.25, 50.0, 77.7][k % 3])
        elif kind == "early_ties":
            t = uniform_times(13.0, 100.0)(rng, n, k)
            t[rng.choice(n, 7, replace=False)] = np.float32(12.75)
        return t
    rng = np.random.default_rng(16)
    tr = Trio()
    tr.run(stream(rng, 4000 if big else 600, times))


def case_size(big, n):
    """n points per scan, not a multiple of the block size; the earliest point past the first IMU pose (chain of 3)."""
    rng = np.random.default_rng(17)
    tr = Trio(oracle_subset=20000)
    tr.run(stream(rng, n, uniform_times(12.5, 100.0), n_moving=3))


def case_pose_cap(big):
    """A 1 kHz IMU on 0.256 s scans: 254 samples per package give the 256 IMU poses the device holds (and match the
    reference); 255 samples are LSD_ERR_CAPACITY, a limit of the device the reference does not have."""
    rng = np.random.default_rng(18)
    n = 3000 if big else 500
    pkgs = stream(rng, n, uniform_times(2.5, 254.0), n_moving=3, hz=1000, period=0.254, off=0.0)
    tr = Trio()
    tr.run(pkgs)
    assert len(tr.r.poses()) == MAX_POSES and len(tr.g.poses()) == MAX_POSES
    last = pkgs[-1]
    beg = last["lidar_end_time"]
    stamps = beg + (np.arange(255) + 1) / 1000.0
    m = dict(lidar_beg_time=beg, lidar_end_time=beg + 0.256, points=cloud(rng, n), time_ms=uniform_times(2.5, 254.0)(rng, n, 0),
             imu=imu_rows(rng, stamps, True), ins_vel=None)
    try:
        tr.g.process(m["imu"], m["lidar_beg_time"], m["lidar_end_time"], m["points"], m["time_ms"], tr.xg, tr.Pg)
    except lsdreg.capi.LsdError as e:
        assert e.status == lsdreg.ERR_CAPACITY, e
    else:
        raise AssertionError("257 IMU poses accepted")
    out_r, _ = tr.r.process(m, tr.xr.copy(), tr.Pr.copy())
    assert len(out_r) == n and len(tr.r.poses()) == MAX_POSES + 1


def case_undistort_off(big):
    """undistort = 0: the forward propagation still runs; the output is the input in input order, and equals the
    reference's sorted cloud mapped back by index."""
    rng = np.random.default_rng(19)
    tr = Trio(undistort=False)
    tr.run(stream(rng, 5000 if big else 600, uniform_times(12.5, 100.0), n_moving=3))


def case_device_path(big):
    """The host path (numpy) and the device path (CUDA torch tensors through lsd_imu_process_dev) give bit-identical
    state, covariance and cloud."""
    import torch
    rng = np.random.default_rng(20)
    pkgs = stream(rng, 6000, uniform_times(12.5, 100.0), n_moving=3)
    tr = Trio()
    h = lsdreg.ImuProcess(ext_R=EXT_R, ext_t=EXT_T)
    xh, Ph = tr.xg.copy(), tr.Pg.copy()
    for m in pkgs:
        st_h, xh, Ph, nh = h.process(m["imu"], m["lidar_beg_time"], m["lidar_end_time"], m["points"], m["time_ms"], xh, Ph)
        tr.step(m, points=torch.from_numpy(m["points"]).cuda(), time_ms=torch.from_numpy(m["time_ms"]).cuda())
        torch.cuda.synchronize()
        assert np.array_equal(xh, tr.xg) and np.array_equal(Ph, tr.Pg)
        if st_h == lsdreg.OK:
            assert np.array_equal(h.cloud(), tr.g.cloud())
    assert tr.n_und >= 3


CASES = {
    "leading_gap_12.5ms": lambda big: case_leading_gap(big, 12.5),
    "leading_gap_57.5ms": lambda big: case_leading_gap(big, 57.5),
    "head_ties": case_head_ties,
    "imu_and_points_past_end": case_past_end,
    "stale_samples_and_gaps": case_stale_gaps,
    "init_paths": case_init_paths,
    "t_negative": lambda big: case_times(big, "negative"),
    "t_negative_zero": lambda big: case_times(big, "negzero"),
    "t_one_time": lambda big: case_times(big, "one_time"),
    "t_mid_ties": lambda big: case_times(big, "mid_ties"),
    "t_early_ties": lambda big: case_times(big, "early_ties"),
    "n_0": lambda big: case_size(big, 0),
    "n_1": lambda big: case_size(big, 1),
    "n_255": lambda big: case_size(big, 255),
    "n_257": lambda big: case_size(big, 257),
    "n_big": lambda big: case_size(big, (1 << 20) + 3 if big else 4099),
    "pose_cap": case_pose_cap,
    "undistort_off": case_undistort_off,
    "device_path": case_device_path,
}
NEEDS_TORCH = {"device_path"}
