"""GPU: the loop-closure detector.  Batched coarse matching equals a separate lsd_reg NDT handle per pair, bit for bit;
detect() equals the CPU restatement of LoopDetector (tests/loop_oracle.py) and finds the planted loop; a scene with no
loop is rejected by the best-score gate; calc_fitness_score counts points beyond the grid search radius; one launch per
LM round."""
import numpy as np
import pytest

import loop_oracle as LO

pytestmark = pytest.mark.gpu

RADIUS, STEP, N_KF = 10.0, 3.0, 22


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


@pytest.fixture(scope="module")
def loop_world():
    """Key frames on a closed circle around the block centre; the last one revisits the start.  Graph estimates drift
    to 1 m / 5 deg by then.  Cloud sizes vary (warp- and thread-shaped fitness)."""
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    truth, est, clouds, accum = [], [], [], []
    L = 2 * np.pi * RADIUS
    for i in range(N_KF):
        s = min(i * STEP, L)
        th = s / RADIUS
        R = synth.rot_from_rpy(0.0, 0.0, th + np.pi / 2)
        t = c0 + np.array([RADIUS * np.cos(th), RADIUS * np.sin(th), 0.0])
        T = _pose(R, t)
        f = s / L
        truth.append(T)
        est.append(_pose(synth.rot_from_rpy(0.0, 0.0, np.deg2rad(5.0) * f) @ R, t + np.array([0.7, 0.7, 0.0]) * f))
        clouds.append(synth.scan64(100 + i, (200, 250, 400)[i % 3], R, t))
        accum.append(s)
    return dict(truth=np.array(truth), est=np.array(est), clouds=clouds, accum=np.array(accum))


@pytest.fixture(scope="module")
def detector(loop_world):
    import lsdreg
    d = lsdreg.LoopDetector()
    for c, a in zip(loop_world["clouds"], loop_world["accum"]):
        d.add_keyframe(c, a)
    return d


def _rot_err(Ra, Rb):
    D = Ra.T @ Rb
    return float(np.linalg.norm(D - D.T) / (2 * np.sqrt(2)))


def test_batched_equals_single(loop_world, detector):
    import lsdreg
    W = loop_world
    new = N_KF - 1
    cands = list(range(0, 12))
    guesses = [LO.initial_guess(W["est"][new], W["est"][k]) for k in cands]
    far = np.eye(4); far[:3, 3] = [500.0, 500.0, 0.0]          # no correspondence anywhere
    cands.append(3); guesses.append(far)
    spin = guesses[5].copy()                                     # 40 degrees off: a long or failed alignment
    spin[:3, :3] = lsdreg.synth.rot_from_rpy(0.0, 0.0, np.deg2rad(40.0)) @ spin[:3, :3]
    cands.append(5); guesses.append(spin.astype(np.float32).astype(np.float64))
    sizes = {W["clouds"][k].shape[0] for k in cands}
    assert len(sizes) >= 3 and min(sizes) < 16384 <= max(sizes)
    m = detector.match(new, cands, np.array(guesses))
    evals = []
    for i, (k, g) in enumerate(zip(cands, guesses)):
        s = lsdreg.Matcher("NDT_CUDA")
        s.set_target(W["clouds"][new]); s.set_source(W["clouds"][k])
        l0 = s.stats()["launches"]
        s.align(g.astype(np.float32))
        evals.append(s.stats()["launches"] - l0)
        T, _ = s.final()
        assert np.array_equal(m["final"][i], T), i
        assert bool(m["converged"][i]) == s.converged and m["iterations"][i] == s.iterations, i
        assert np.array_equal(m["iteration_logs"][i], s.iteration_log()), i
        fs = s.fitness(25.0)
        assert m["fitness"][i] == fs, i
    assert not m["converged"][12]
    assert m["converged"][:12].sum() >= 2
    # one launch per round; rounds = the most cost evaluations any one candidate needed, not their sum
    assert m["rounds"] == max(evals) < sum(evals)
    again = detector.match(new, cands, np.array(guesses))      # target maps already built: rounds + one fitness launch
    assert again["launches"] == again["rounds"] + 1
    assert np.array_equal(again["final"], m["final"])


def test_detect_matches_oracle_and_finds_the_loop(loop_world, detector):
    W = loop_world
    new = [N_KF - 2, N_KF - 1]
    kfs = list(range(N_KF - 2))
    detector.last_edge_accum_distance = 0.0
    loops = detector.detect(W["est"], kfs, new)
    reps = detector.reports()
    o = LO.OracleLoopDetector(W["clouds"], W["accum"])
    oloops, oreps = o.detect(W["est"], kfs, new)
    names = ["skipped", "no_candidates", "coarse_reject", "gicp_diverged", "gicp_reject", "found"]
    assert [names[r["decision"]] for r in reps] == [r["decision"] for r in oreps]
    for r, orr in zip(reps, oreps):
        assert r["n_candidates"] == orr.get("n_candidates", 0)
        if "best_slot" in orr:
            assert r["best_slot"] == orr["best_slot"]
            np.testing.assert_allclose(r["best_score"], orr["best_score"], rtol=1e-5)
    assert len(loops) == len(oloops) >= 1
    for g, ol in zip(loops, oloops):
        assert (g["key1"], g["key2"]) == (ol["key1"], ol["key2"])
        assert np.abs(g["relpose"][:3, 3] - ol["relpose"][:3, 3]).max() < 1e-4
        assert _rot_err(g["relpose"][:3, :3].astype(np.float64), ol["relpose"][:3, :3].astype(np.float64)) < 1e-5
        np.testing.assert_allclose(g["coarse_score"], ol["coarse_score"], rtol=1e-5)
        np.testing.assert_allclose(g["score"], ol["score"], rtol=1e-5)
        np.testing.assert_allclose(g["information"], ol["information"], rtol=1e-6)
        # the planted loop: relpose = truth_new^-1 * truth_candidate
        Tt = np.linalg.inv(W["truth"][g["key1"]]) @ W["truth"][g["key2"]]
        assert np.abs(g["relpose"][:3, 3] - Tt[:3, 3]).max() < 0.05
    assert detector.last_edge_accum_distance == W["accum"][loops[-1]["key1"]]


def test_no_loop_in_another_block():
    """Candidates whose clouds look at another block from another spot: nothing aligns, the best-score gate rejects."""
    import lsdreg
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    c1 = synth.block_center(1, 0) + np.array([30.0, 12.0, 0.0])
    d = lsdreg.LoopDetector()
    clouds, accum, poses = [], [], []
    for i in range(4):
        clouds.append(synth.scan64(300 + i, 250, np.eye(3), c1 + np.array([2.0 * i, 0.0, 0.0]), bi=1))
        accum.append(2.5 * i); poses.append(_pose(np.eye(3), c0 + np.array([2.0 * i, 0.0, 0.0])))
    clouds.append(synth.scan64(310, 250, np.eye(3), c0)); accum.append(40.0); poses.append(_pose(np.eye(3), c0))
    for c, a in zip(clouds, accum):
        d.add_keyframe(c, a)
    assert d.detect(np.array(poses), [0, 1, 2, 3], [4]) == []
    rep = d.reports()[0]
    assert rep["decision"] == lsdreg.LOOP_COARSE_REJECT and rep["n_candidates"] == 4
    assert rep["best_score"] > 2 * 1.5
    o = LO.OracleLoopDetector(clouds, accum)
    oloops, oreps = o.detect(np.array(poses), [0, 1, 2, 3], [4])
    assert oloops == [] and oreps[0]["decision"] == "coarse_reject" and oreps[0]["best_slot"] == rep["best_slot"]


@pytest.mark.parametrize("n_az", [200, 300])
def test_information_fitness_counts_far_points(n_az):
    """calc_fitness_score (max_range = DBL_MAX) counts points with nothing within the 32 m grid search radius."""
    import lsdreg
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    tgt = synth.scan64(401, 250, np.eye(3), c0)
    src = synth.scan64(402, n_az, np.eye(3), c0 + np.array([0.5, 0.0, 0.0]))
    src[::50, 2] += 60.0                      # > 50 m above anything in the target
    d = lsdreg.LoopDetector()
    a = d.add_keyframe(tgt, 0.0); b = d.add_keyframe(src, 0.0)
    T = np.eye(4, dtype=np.float32); T[0, 3] = 0.5
    score, n = d.fitness(a, b, T)
    oscore, on = LO.calc_fitness_score(tgt, src, T)
    assert n == on == src.shape[0]
    np.testing.assert_allclose(score, oscore, rtol=1e-6)
    s25, n25 = d.fitness(a, b, T, 25.0)       # getFitnessScore(25): the far points drop out
    assert n25 < n and s25 < score
