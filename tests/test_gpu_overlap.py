"""GPU: the overlap detector of map merging (lsd_overlap_*).  The filtered calc_fitness_score equals a brute-force numpy
version (counts exact, score to 1e-12), also on a target whose point map refuses points and at a pose where nothing
counts; the batched NDT of pairs spanning several new key frames equals lsd_reg's single-pair kernels on the same tables
bit for bit, and separate lsd_reg NDT handles whenever they rebuild the same table, in one cost launch per round; detect()
over two fragments equals the restatement of OverlapDetector (tests/overlap_oracle.py), finds the planted overlaps,
rejects through the prescreen and the final gate, and accumulates keyframes[0] for a connection outside the loaded map;
detect releases its target tables when it returns; an empty filtered target still reports the kept source points."""
import numpy as np
import pytest

import overlap_oracle as OO

pytestmark = pytest.mark.gpu

N_AZ = 160          # x 64 beams: ~10 k points per key frame
NEW0 = 1000         # graph ids of the new map


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _chain(ids):
    return [(a, b) for a, b in zip(ids[:-1], ids[1:])]


@pytest.fixture(scope="module")
def world():
    """Loaded map: 10 key frames every 3 m through block (0, 0), ids 0..9, a chain.  New map: a chain of ids 1000..1039;
    fragment A = ids 1010..1015 (four 0.5 m beside loaded key frames 2..5, turned, the second with 70 % of its points
    thrown up to 3 m, then two in block (1, 0)), fragment B = ids 1030..1033 over loaded key frames 2..5 again, the last
    with a pose estimate 6 m / 25 deg off (nothing passes its prescreen)."""
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    rng = np.random.default_rng(3)
    clouds, poses, ids = [], [], []
    for i in range(10):
        R = synth.rot_from_rpy(0.0, 0.0, 0.15 * i)
        t = c0 + np.array([-15.0 + 3.0 * i, 1.0, 0.0])
        clouds.append(synth.scan64(300 + i, N_AZ, R, t)); poses.append(_pose(R, t)); ids.append(i)
    frag = {}
    for name, base, seed in (("A", 1010, 400), ("B", 1030, 500)):
        frag[name] = []
        for j, i in enumerate((2, 3, 4, 5)):
            R = synth.rot_from_rpy(0.0, 0.0, 0.15 * i + 0.4 + 0.1 * j)
            t = poses[i][:3, 3] + np.array([0.4, -0.5 if name == "A" else 0.6, 0.0])
            c = synth.scan64(seed + j, N_AZ, R, t)
            T = _pose(R, t)
            if name == "A" and j == 1:
                m = rng.random(len(c)) < 0.7
                c = c.copy(); c[m, :3] += rng.uniform(-3.0, 3.0, (int(m.sum()), 3)).astype(np.float32)
            if name == "B" and j == 3:
                T = _pose(synth.rot_from_rpy(0.0, 0.0, np.deg2rad(25.0)) @ R, t + np.array([6.0, 0.0, 0.0]))
            frag[name].append(len(clouds)); clouds.append(c); poses.append(T); ids.append(base + j)
    c1 = synth.block_center(1, 0)
    for j in range(2):
        R = synth.rot_from_rpy(0.0, 0.0, 0.5 * j)
        t = c1 + np.array([5.0 * j - 3.0, -6.0, 0.0])
        frag["A"].append(len(clouds)); clouds.append(synth.scan64(600 + j, N_AZ, R, t, bi=1)); poses.append(_pose(R, t))
        ids.append(1014 + j)
    edges = _chain(list(range(10))) + _chain(list(range(NEW0, NEW0 + 40)))
    return dict(clouds=clouds, poses=np.array(poses), ids=ids, kfs=list(range(10)), A=frag["A"], B=frag["B"], edges=edges)


@pytest.fixture(scope="module")
def detector(world):
    import lsdreg
    d = lsdreg.OverlapDetector()
    for c, i in zip(world["clouds"], world["ids"]):
        d.add_keyframe(c, i)
    return d


def _dense_target(world):
    """A key frame plus 2 000 points inside one 0.1 m cube: more than one point-map voxel holds (896)."""
    rng = np.random.default_rng(9)
    blob = np.zeros((2000, 4), np.float32)
    blob[:, :3] = np.array([6.0, 4.0, 1.5], np.float32) + rng.uniform(0, 0.1, (2000, 3)).astype(np.float32)
    return np.concatenate([world["clouds"][3], blob], 0)


def test_filtered_fitness_against_brute_force(world, detector):
    import lsdreg
    W = world
    dense = lsdreg.OverlapDetector()
    s_dense = dense.add_keyframe(_dense_target(W), 77)
    s_src = dense.add_keyframe(W["clouds"][W["A"][1]], 78)
    cases = [(detector, W["A"][0], 2, OO.guess(W["poses"][W["A"][0]], W["poses"][2]), 1.0, W["clouds"][W["A"][0]], W["clouds"][2]),
             (detector, W["A"][2], 4, OO.guess(W["poses"][W["A"][2]], W["poses"][4]), 25.0, W["clouds"][W["A"][2]], W["clouds"][4]),
             (dense, s_dense, s_src, OO.guess(W["poses"][3], W["poses"][W["A"][1]]), 25.0, _dense_target(W), W["clouds"][W["A"][1]])]
    far = np.eye(4, dtype=np.float32); far[:3, 3] = [0.0, 0.0, 60.0]   # every kept source point 50+ m above the target
    cases.append((detector, 0, 1, far, 1.0, W["clouds"][0], W["clouds"][1]))
    low = W["clouds"][4].copy(); low[:, 2] = -1.0                          # nothing passes the filter: an empty target
    s_low = dense.add_keyframe(low, 79)
    cases.append((dense, s_low, s_src, OO.guess(W["poses"][3], W["poses"][W["A"][1]]), 25.0, low, W["clouds"][W["A"][1]]))
    for k, (d, t, s, T, mr, tc, sc) in enumerate(cases):
        got = d.fitness(t, s, T, mr)
        score, ratio, nr, nf = OO.calc_fitness_score(tc, sc, T, mr)
        assert got["n_counted"] == nr and got["n_filtered"] == nf, k
        if nr == 0:
            assert got["score"] == OO.DBL_MAX and got["inlier_ratio"] == 0.0, k
        else:
            np.testing.assert_allclose(got["score"], score, rtol=1e-12)
            assert got["inlier_ratio"] == ratio
        assert got["target_incomplete"] == (k == 2), k
    assert OO.calc_fitness_score(W["clouds"][0], W["clouds"][1], far, 1.0)[2] == 0
    assert OO.calc_fitness_score(low, W["clouds"][W["A"][1]], cases[-1][3], 25.0)[3] > 0   # kept source points, none counted


def test_batched_equals_single(world, detector):
    import lsdreg
    W = world
    new = [W["A"][0], W["A"][0], W["A"][2], W["A"][2], W["A"][3], W["B"][0]]
    cand = [2, 3, 4, 5, 5, 2]
    G = [OO.guess(W["poses"][n], W["poses"][c]).astype(np.float64) for n, c in zip(new, cand)]
    far = np.eye(4); far[:3, 3] = [500.0, 500.0, 0.0]
    new.append(W["A"][2]); cand.append(3); G.append(far)
    m = detector.match(new, cand, np.array(G))
    ser = detector.match(new, cand, np.array(G), serial=True)   # lsd_reg's single-pair kernels on the same tables
    for k in ("final", "converged", "iterations", "fitness"):
        assert np.array_equal(m[k], ser[k]), k
    for lb, ls in zip(m["iteration_logs"], ser["iteration_logs"]):
        assert np.array_equal(lb, ls)
    evals = [detector.match([n], [c], np.array([g]), serial=True)["rounds"] for n, c, g in zip(new, cand, G)]
    assert ser["rounds"] == sum(evals)
    for i, (n, c, g) in enumerate(zip(new, cand, G)):
        # a separate lsd_reg NDT handle builds its own table, and the double atomic sums of a table build can differ in
        # the last bits from build to build (two separate handles can disagree too): the pair equals one of a few
        # separate builds bit for bit, or, when none of them rebuilt this handle's table, agrees to 1e-9
        for _ in range(4):
            s = lsdreg.Matcher("NDT_CUDA")
            s.set_target(W["clouds"][n]); s.set_source(W["clouds"][c])
            l0 = s.stats()["launches"]
            s.align(g.astype(np.float32))
            T, _ = s.final()
            if np.array_equal(m["final"][i], T):
                break
        assert bool(m["converged"][i]) == s.converged and m["iterations"][i] == s.iterations, i
        if not np.array_equal(m["final"][i], T):
            np.testing.assert_allclose(m["final"][i], T, rtol=0, atol=1e-9)
            continue
        assert s.stats()["launches"] - l0 == evals[i], i
        assert np.array_equal(m["iteration_logs"][i], s.iteration_log()), i
        if s.converged:
            assert m["fitness"][i] == s.fitness(25.0), i
    assert not m["converged"][-1] and m["converged"][:-1].sum() >= 4
    assert m["rounds"] == max(evals) < sum(evals)
    again = detector.match(new, cand, np.array(G))          # tables built: one launch per round + one fitness launch
    assert again["launches"] == again["rounds"] + 1
    assert np.array_equal(again["final"], m["final"])


def _rot_err(Ra, Rb):
    D = Ra.T @ Rb
    return float(np.linalg.norm(D - D.T) / (2 * np.sqrt(2)))


NAMES = ["no_candidates", "no_match", "gicp_diverged", "gicp_reject", "found"]


def _compare(d, o, W, new, edges):
    got = d.detect(W["poses"], W["kfs"], new, edges)
    reps = d.reports()
    oov, oreps = o.detect(W["poses"], W["kfs"], new, edges)
    assert [NAMES[r["decision"]] for r in reps] == [r["decision"] for r in oreps]
    for r, orr, ns in zip(reps, oreps, new):
        assert list(d.find_candidates(W["poses"], W["kfs"], ns, edges)) == orr["candidates"]
        assert r["n_candidates"] == orr["n_candidates"] and r["n_prescreened"] == orr["n_prescreened"]
        assert r["best_slot"] == orr["best_slot"] and r["n_accum"] == orr["n_accum"]
        if orr["best_slot"] >= 0:
            np.testing.assert_allclose(r["best_score"], orr["best_score"], rtol=1e-5)
        if "score" in orr:
            np.testing.assert_allclose(r["score"], orr["score"], rtol=1e-5, atol=1e-5)
    assert len(got) == len(oov)
    for g, og in zip(got, oov):
        assert (g["key1"], g["key2"]) == (og["key1"], og["key2"])
        assert np.abs(g["relpose"][:3, 3] - og["relpose"][:3, 3]).max() < 1e-4
        assert _rot_err(g["relpose"][:3, :3], og["relpose"][:3, :3]) < 1e-5
        np.testing.assert_allclose(g["score"], og["score"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(g["coarse_score"], og["coarse_score"], rtol=1e-5)
    return got, reps, oreps


def test_detect_two_fragments_matches_oracle(world, detector):
    W = world
    o = OO.OracleOverlapDetector(W["clouds"], W["ids"])
    edges = list(W["edges"])
    got_a, reps_a, _ = _compare(detector, o, W, W["A"], edges)
    dec_a = [NAMES[r["decision"]] for r in reps_a]
    assert dec_a[0] == dec_a[2] == dec_a[3] == "found"                          # the planted overlaps
    assert dec_a[1] == "gicp_reject"                                            # the scattered cloud
    assert dec_a[4] in ("no_candidates", "no_match") and dec_a[5] in ("no_candidates", "no_match")   # another block
    st = detector.stats()
    assert st["rounds"] >= 1 and st["launches"] > st["rounds"]
    # the caller's graph_add_edge of every overlap, then the second fragment
    edges += [(W["ids"][g["key1"]], W["ids"][g["key2"]]) for g in got_a]
    got_b, reps_b, oreps_b = _compare(detector, o, W, W["B"], edges)
    dec_b = [NAMES[r["decision"]] for r in reps_b]
    assert dec_b[3] == "no_match" and reps_b[3]["n_candidates"] > 0 and reps_b[3]["n_prescreened"] == 0
    assert "found" in dec_b
    # keyframe_id_map's default 0: a best candidate connected to a new-map key frame of fragment A accumulates
    # keyframes[0]'s cloud for that connection
    linked = {g["key1"] for g in got_a}
    quirk = [r for r in reps_b if r["best_slot"] in linked]
    assert quirk
    for r in quirk:
        b = r["best_slot"]
        conn = OO.connections(edges)[W["ids"][b]]
        want = len(W["clouds"][b]) + sum(len(W["clouds"][c if c < 10 else 0]) for c in conn)
        assert r["n_accum"] == want
        assert any(c >= NEW0 for c in conn)


def test_detect_releases_its_tables(world):
    """Every new key frame is a target in one fragment only: detect hands its tables back when it returns, and the next
    call reuses the buffers, so device memory follows one fragment, not the merge."""
    import lsdreg
    W = world
    d = lsdreg.OverlapDetector()
    for c, i in zip(W["clouds"], W["ids"]):
        d.add_keyframe(c, i)
    d.detect(W["poses"], W["kfs"], W["A"], W["edges"])
    first = d.stats()
    assert first["targets_held"] == 0 and 1 <= first["target_buffers"] <= len(W["A"])
    for frag in ("B", "A", "B"):
        d.detect(W["poses"], W["kfs"], W[frag], W["edges"])
        st = d.stats()
        assert st["targets_held"] == 0 and st["target_buffers"] <= len(W["A"])
