"""CPU: the restated floor detector of tests/floor_oracle.py — its generator against C++ std::mt19937 (the engine
boost::mt19937 is), lsd_ransac_replay against the restated stop rule, and the whole detector on synthetic scenes with a
known plane and at each failure gate."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import floor_oracle as FO
import lsdreg

_HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def mt_harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mt") / "libmt_host_harness.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-o", out,
                           os.path.join(_HERE, "mt_host_harness.cpp")])
    L = C.CDLL(out)
    L.mt19937_outputs.argtypes = [C.c_uint32, C.c_void_p, C.c_int]
    return L


def test_generator_equals_std_mt19937(mt_harness):
    n = 1_000_000
    ref = np.zeros(n, np.uint32)
    mt_harness.mt19937_outputs(12345, ref.ctypes.data, n)
    g = FO.MT19937(12345)
    mine = g.outputs(n)
    assert np.array_equal(mine, ref)
    # next() and outputs() walk the same stream
    g2 = FO.MT19937(12345)
    assert [g2.next() for _ in range(1500)] == [int(v) for v in ref[:1500]]
    # the C++ standard's check value: the 10000th output of a default-seeded (5489) mt19937
    assert int(FO.MT19937(5489).outputs(10000)[-1]) == 4123659995

def _replay_both(counts, flags, n_points, p=0.99, max_iter=10000):
    g = lsdreg.ransac_replay(counts, flags, n_points, p, max_iter)
    o = FO.stop_rule(counts, flags, n_points, p, max_iter)
    assert (g["consumed"], g["best"], g["iterations"], g["skipped"]) == (o["consumed"], o["best"], o["iterations"], o["skipped"]), (g, o)
    return g


def test_replay_equals_the_restated_stop_rule_on_random_sequences():
    rng = np.random.default_rng(3)
    ended = 0
    for trial in range(400):
        n_points = int(rng.integers(3, 50000))
        n = int(rng.integers(1, 600))
        kind = trial % 5
        if kind == 0:     # ordinary counts
            counts = rng.integers(0, n_points + 1, n)
        elif kind == 1:   # ties: few distinct values
            counts = rng.choice(rng.integers(0, n_points + 1, 3), n)
        elif kind == 2:   # w -> 0
            counts = rng.integers(0, 3, n)
        elif kind == 3:   # w = 1 somewhere
            counts = rng.integers(0, n_points + 1, n); counts[rng.integers(0, n)] = n_points
        else:             # slowly growing best: long runs
            counts = np.minimum(np.cumsum(rng.integers(0, 3, n)), n_points)
        flags = np.where(rng.random(n) < 0.1, 0, 1)
        if trial % 7 == 0:
            flags[rng.integers(0, n)] = -1
        max_iter = int(rng.choice([10000, 50, 5, 0]))
        g = _replay_both(counts, flags, n_points, 0.99, max_iter)
        ended += g["consumed"] >= 0
    assert ended > 100


def test_replay_edges():
    # w = 1 on the first hypothesis: k = log(0.01) / log(eps) < 1, one iteration
    g = _replay_both([100], [1], 100)
    assert g["consumed"] == 1 and g["best"] == 0 and g["iterations"] == 1
    # a tie keeps the earlier hypothesis
    g = _replay_both([10, 10, 10] * 50, [1, 1, 1] * 50, 20)
    assert g["best"] == 0
    # skipped hypotheses count without iterating; the 10 x max_iterations cut
    g = _replay_both([0] * 60, [0] * 60, 1000, 0.99, 5)
    assert g["consumed"] == 50 and g["skipped"] == 50 and g["iterations"] == 0 and g["best"] == -1
    # the max_iterations cut: iterations > max after the increment
    g = _replay_both([1] * 20, [1] * 20, 10 ** 6, 0.99, 7)
    assert g["consumed"] == 8 and g["iterations"] == 8
    # no sample could be drawn
    g = _replay_both([5, 0, 7], [1, -1, 1], 100)
    assert g["consumed"] == 2 and g["best"] == 0 and g["iterations"] == 1
    # not ended: more hypotheses needed
    g = _replay_both([1, 1], [1, 1], 10 ** 6)
    assert g["consumed"] == -1


def _plane_ok(c, roll_deg, ground_z, tol=0.02):
    n = FO.rot_x(roll_deg) @ np.array([0.0, 0.0, 1.0])
    assert c[2] >= 0
    assert np.abs(c[:3] - n).max() < tol, (c, n)
    assert abs(c[3] - (-ground_z)) < 0.05, c


@pytest.mark.parametrize("preset,ground_z", [(FO.MAPPING, -1.8), (FO.GROUND, -0.3), (FO.RENDER, -0.3)])
def test_restated_detector_recovers_the_plane(preset, ground_z):
    p = FO.default_params(preset)
    for roll in (0.0, 4.0):
        pts = FO.scene(11, n_ground=15000, ground_z=ground_z, roll_deg=roll, radius=12.0, walls=2)
        r = FO.detect(pts, p)
        assert r["found"] and r["reason"] == FO.FOUND, r["reason"]
        _plane_ok(r["coeffs"], roll, ground_z)
        rs = r["ransac"]
        assert rs["counts"][rs["best"]] == r["inliers"].shape[0] >= p["floor_pts_thresh"]


def test_restated_detector_gates():
    p = FO.default_params(FO.MAPPING)
    assert FO.detect(np.zeros((0, 4), np.float32), p)["reason"] == FO.EMPTY
    # rolled 14 deg: the normals pass the 20 deg filter, the plane fails the 10 deg check
    r = FO.detect(FO.scene(5, n_ground=15000, roll_deg=14.0, radius=12.0), p)
    assert r["reason"] == FO.NOT_VERTICAL and not r["found"]
    # ground below the clip band
    r = FO.detect(FO.scene(5, n_ground=15000, ground_z=-3.0, radius=12.0), p)
    assert r["reason"] == FO.FEW_CANDIDATES
    # two parallel planes of 800 points each: 1600 candidates, the best plane holds 800 inliers
    q = FO.default_params(FO.GROUND)
    a = FO.scene(2, n_ground=800, ground_z=-0.3, radius=6.0)
    b = FO.scene(3, n_ground=800, ground_z=0.4, radius=6.0)
    r = FO.detect(np.concatenate([a, b]), q)
    assert r["reason"] == FO.FEW_INLIERS, r["reason"]
    # exactly collinear candidates (dyadic steps, so the three ratios are equal in float): every draw fails isSampleGood,
    # 1000 redraws, no model
    q = dict(FO.default_params(FO.GROUND), use_normal_filtering=0, floor_pts_thresh=3)
    k = np.arange(40, dtype=np.float32)
    line = np.stack([k / 8, k / 4, -k / 32, k], 1).astype(np.float32)
    r = FO.detect(line, q)
    assert r["reason"] == FO.NO_MODEL and r["ransac"]["flags"].tolist() == [-1]


def test_restated_normals_of_a_plane():
    """On a noiseless tilted plane every normal is the plane's (up to the viewpoint sign) and curvature ~0."""
    rng = np.random.default_rng(1)
    xy = rng.uniform(-3, 3, (2000, 2))
    n = FO.rot_x(7.0) @ np.array([0.0, 0.0, 1.0])
    z = (-1.5 - n[0] * xy[:, 0] - n[1] * xy[:, 1]) / n[2]
    xyz = np.stack([xy[:, 0], xy[:, 1], z], 1).astype(np.float32)
    nrm, cov6, nbr = FO.normals(xyz)
    assert (nbr[:, 0] == np.arange(2000)).all()   # the point itself first (d2 = 0)
    dots = np.abs(nrm[:, :3].astype(np.float64) @ n)
    assert dots.min() > 1 - 1e-4
    assert np.nanmax(nrm[:, 3]) < 1e-4
    # the viewpoint flip: every normal points at the sensor (origin) side, i.e. upward for a plane below it
    assert (nrm[:, :3].astype(np.float64) @ n > 0).all()
    assert math.isclose(float(np.median(np.abs(FO.normal_nz(nrm)))), n[2], rel_tol=1e-4)
