"""CPU: the host half of the overlap detector of map merging (lsd_overlap_find_candidates, the guesses) against the
restatement of OverlapDetector (tests/overlap_oracle.py) on random trajectories and graphs built to reach the edges of
get_connection_count: the level cap, a disconnected pair, an id pushed twice into one level, a candidate exactly 30 m away,
fewer key frames than the 10-NN asks for."""
import numpy as np
import pytest

import overlap_oracle as OO


def _pose(yaw, t):
    T = np.eye(4)
    c, s = np.cos(yaw), np.sin(yaw)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = t
    return T


def _world(seed, n_old=30, n_new=12, spread=40.0):
    rng = np.random.default_rng(seed)
    poses = [_pose(rng.uniform(-np.pi, np.pi), rng.uniform(-spread, spread, 3) * [1, 1, 0.05]) for _ in range(n_old + n_new)]
    ids = list(range(n_old)) + list(range(500, 500 + n_new))
    return np.array(poses), ids


def _chain(ids):
    return [(a, b) for a, b in zip(ids[:-1], ids[1:])]


def _check(poses, ids, kfs, new_slots, edges):
    import lsdreg
    for ns in new_slots:
        got = lsdreg.overlap_find_candidates(poses, ids, kfs, ns, edges)
        want = OO.find_candidates(poses, ids, kfs, ns, edges)
        assert list(got) == want, (ns, list(got), want)


@pytest.mark.parametrize("seed", range(6))
def test_candidates_random(seed):
    poses, ids = _world(seed)
    rng = np.random.default_rng(seed + 100)
    old, new = ids[:30], ids[30:]
    edges = _chain(old) + _chain(new)
    # a few overlap edges between the maps and random shortcuts inside the old one
    for _ in range(4):
        edges.append((int(rng.choice(old)), int(rng.choice(new))))
    for _ in range(3):
        edges.append(tuple(int(v) for v in rng.choice(old, 2, replace=False)))
    _check(poses, ids, list(range(30)), list(range(30, 42)), edges)


def test_level_cap_and_disconnected():
    poses, ids = _world(7, n_old=12, n_new=4, spread=10.0)
    old, new = ids[:12], ids[12:]
    # disconnected maps: the count is the levels of the new key frame's component (a chain of 4, then a chain of 14)
    _check(poses, ids, list(range(12)), list(range(12, 16)), _chain(old) + _chain(new))
    long_chain = new + [900 + i for i in range(12)]
    _check(poses, ids, list(range(12)), list(range(12, 16)), _chain(old) + _chain(long_chain))
    # connected at distance 9, 10 and 11 along the graph
    for hops in (8, 9, 10):
        path = [new[0]] + [700 + i for i in range(hops)] + [old[0]]
        _check(poses, ids, list(range(12)), [12], _chain(old) + _chain(path))


def test_repeated_queue_entries():
    """A triangle: the BFS pushes a node again from a node of its own level; with the target unreachable that adds a level."""
    poses, ids = _world(8, n_old=8, n_new=3, spread=8.0)
    old, new = ids[:8], ids[8:]
    tri = [(new[0], new[1]), (new[0], new[2]), (new[1], new[2])]
    for extra in range(0, 10):
        tail = [new[2]] + [600 + i for i in range(extra)]
        edges = _chain(old) + tri + _chain(tail)
        _check(poses, ids, list(range(8)), [8, 9, 10], edges)
    # the literal queue and a plain BFS disagree here, which is what the restatement reproduces
    conn = OO.connections(tri)
    assert OO.connection_count(conn, new[0], -1, 10) == 3


def test_exactly_30m_and_few_keyframes():
    poses = np.array([_pose(0.0, [30.0, 0.0, 0.0]), _pose(0.0, [29.999998, 0.0, 0.0]), _pose(0.0, [0.0, 30.0, 0.0]),
                      _pose(0.0, [0.0, 0.0, 0.0])])
    ids = [10, 11, 12, 99]
    kfs = [0, 1, 2]                     # fewer than 10
    edges = _chain([99] + [900 + i for i in range(12)])   # the new key frame's component reaches the level cap
    got = list(__import__("lsdreg").overlap_find_candidates(poses, ids, kfs, 3, edges))
    assert got == OO.find_candidates(poses, ids, kfs, 3, edges) == [1]   # exactly 30 m is not < 30 m
    # the same key frame id and an already connected id are skipped
    ids2 = [99, 11, 12, 99]
    _check(poses, ids2, kfs, [3], edges + [(99, 12)])
    _check(poses, ids, [], [3], [])


def test_guess_bits():
    import lsdreg
    rng = np.random.default_rng(5)
    for _ in range(50):
        from lsdreg import synth
        Ta = np.eye(4); Ta[:3, :3] = synth.rot_from_rpy(*rng.uniform(-0.2, 0.2, 2), rng.uniform(-3, 3)); Ta[:3, 3] = rng.uniform(-500, 500, 3)
        Tb = np.eye(4); Tb[:3, :3] = synth.rot_from_rpy(*rng.uniform(-0.2, 0.2, 2), rng.uniform(-3, 3)); Tb[:3, 3] = rng.uniform(-500, 500, 3)
        g = lsdreg.overlap_guess(Ta, Tb)
        assert np.array_equal(g.view(np.uint32), OO.guess(Ta, Tb).view(np.uint32))
        f = lsdreg.overlap_finetune_guess(g)
        assert np.array_equal(f.view(np.uint32), OO.finetune_guess(g).view(np.uint32))
        assert np.allclose(f.astype(np.float64) @ g.astype(np.float64), np.eye(4), atol=1e-2)   # float translations of up to ~1 km


def test_slots_checked():
    """find_candidates indexes poses and ids by slot: a slot outside them is refused, not read."""
    import lsdreg
    poses, ids = _world(9, n_old=5, n_new=1)
    with pytest.raises(lsdreg.LsdError):
        lsdreg.overlap_find_candidates(poses, ids, [0, 1, 9], 5, [])
    with pytest.raises(lsdreg.LsdError):
        lsdreg.overlap_find_candidates(poses, ids, [0, 1], 6, [])
    with pytest.raises(lsdreg.LsdError):
        lsdreg.overlap_find_candidates(poses, ids, [-1], 5, [])
