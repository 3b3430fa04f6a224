"""CPU: the loop detector's host logic — find_candidates, the initial guesses and the information-matrix weights — against
the restatement of loop_detector.hpp / information_matrix_calculator.cpp in tests/loop_oracle.py."""
import numpy as np

import lsdreg
import loop_oracle as LO


def _trajectory(seed, n=40, step=2.5, radius=12.0, noise_rot=0.0):
    """Key frames every `step` m on a circle, graph estimates with a seeded drift; rotations optionally a little off SO(3)."""
    rng = np.random.default_rng(seed)
    accum = np.arange(n) * step
    poses = np.tile(np.eye(4), (n, 1, 1))
    for i in range(n):
        th = accum[i] / radius
        poses[i, :3, :3] = lsdreg.synth.rot_from_rpy(*rng.normal(0, 0.02, 2), th + np.pi / 2)
        poses[i, :3, 3] = [radius * np.cos(th), radius * np.sin(th), rng.normal(0, 0.3)]
        if noise_rot:
            poses[i, :3, :3] += rng.normal(0, noise_rot, (3, 3))
    return poses, accum


def _check(poses, accum, kfs, new, last_edge=0.0):
    c, G = lsdreg.find_loop_candidates(poses, accum, kfs, new, last_edge)
    oc = LO.find_candidates(poses, accum, kfs, new, last_edge)
    assert list(c) == oc
    for k, g in zip(c, G):
        og = LO.initial_guess(poses[new], poses[k])
        np.testing.assert_allclose(g, og, rtol=0, atol=2e-6)
        assert g[2, 3] == 0.0
        assert np.array_equal(g, g.astype(np.float32).astype(np.float64))   # a float matrix, as the reference's
    return list(c)


def test_candidates_and_guesses_match_oracle():
    for seed in range(6):
        poses, accum = _trajectory(seed, noise_rot=1e-4 if seed % 2 else 0.0)
        for new in (10, 25, 33, 39):
            _check(poses, accum, list(range(new)), new)
            _check(poses, accum, list(range(new)), new, last_edge=accum[new] - 20.0)


def test_guess_normalises_a_non_orthonormal_estimate():
    poses, _ = _trajectory(3)
    Tn, Tc = poses[30].copy(), poses[2].copy()
    Tc[:3, :3] *= 1.001            # a graph estimate whose rotation block drifted off SO(3)
    Tc[0, 1] += 2e-4
    g = lsdreg.find_loop_candidates(np.stack([Tc, Tn]), [0.0, 60.0], [0], 1)[1][0]
    np.testing.assert_allclose(g, LO.initial_guess(Tn, Tc), atol=2e-6)
    R = g[:3, :3]
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-6           # orthonormal again, not the raw product
    raw = np.linalg.inv(Tn) @ Tc
    assert np.abs(raw[:3, :3] - R).max() > 1e-4


def test_threshold_edges():
    """Distances exactly at the 2 m / 25 m / 15 m thresholds: the reference's < and > comparisons decide."""
    n = 6
    poses = np.tile(np.eye(4), (n, 1, 1))
    accum = np.array([0.0, 2.0, 3.9, 10.0, 20.0, 25.0 + 10.0])
    poses[:, 0, 3] = [0.0, 1.0, 2.0, 15.0, 15.0 + 1e-9, 0.0]
    kfs = list(range(n - 1))
    # slot 3: accum 25 back exactly (not < 25), 15 m away exactly (not > 15) -> kept; slot 4: 15 m + 1e-9 -> dropped
    # slot 1: 2 m after slot 0 exactly (not < 2) -> kept; slot 2: 1.9 m after slot 1 -> dropped
    c = _check(poses, accum, kfs, n - 1)
    assert c == [0, 1, 3]
    # last-edge gate: exactly 15 m since the last loop passes, 14.999 does not
    assert _check(poses, accum, kfs, n - 1, last_edge=accum[-1] - 15.0) == [0, 1, 3]
    assert _check(poses, accum, kfs, n - 1, last_edge=accum[-1] - 14.999) == []


def test_last_edge_gate_across_two_detect_calls():
    """detect's second call sees the last_edge_accum_distance the first call's loop left (loop_detector.hpp:60,216)."""
    poses, accum = _trajectory(1)
    kfs = list(range(30))
    first = _check(poses, accum, kfs, 30)
    assert first
    edge = accum[30]                                    # a loop was accepted at new key frame 30
    assert _check(poses, accum, list(range(31)), 31, last_edge=edge) == []      # 2.5 m later: gated
    assert _check(poses, accum, list(range(37)), 37, last_edge=edge) != []      # 17.5 m later: open again


def test_information_matrix_weights():
    for f in (0.0, 1e-3, 0.05, 0.3, 0.5, 1.4, 3.0, 50.0, 1e300):
        got = lsdreg.loop_information_matrix(f)
        np.testing.assert_array_equal(got, LO.information_matrix(f))
    inf = lsdreg.loop_information_matrix(0.5)
    assert abs(1.0 / inf[0, 0] - np.float32(25.0)) < 1e-5 and abs(1.0 / inf[3, 3] - np.float32(0.04)) < 1e-7
