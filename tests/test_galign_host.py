"""CPU: the candidate merge of global alignment (global_alignment.hpp:207-227) — detectCandidateMatch's threshold, one entry per
database index, the smaller float sc_dist wins, the first seen on a tie, ascending index — against the restatement in
tests/galign_oracle.py, on the layout lsd_sc_query returns ([n_off, 10] candidates, -1 padded)."""
import numpy as np

import galign_oracle as GO
import lsdreg


def _check(idx, dist, shift, n_cand, thres=0.30):
    gi, gd, gy = lsdreg.galign_merge_candidates(idx, dist, shift, n_cand, thres)
    per = [GO.candidates_from_query(idx[o], dist[o], shift[o], n_cand[o], thres) for o in range(len(n_cand))]
    om = GO.merge_candidates(per)
    assert list(gi) == [m[0] for m in om]
    assert np.array_equal(gd, np.array([m[1] for m in om], np.float32))
    assert np.array_equal(gy, np.array([m[2] for m in om], np.float32))
    assert list(gi) == sorted(set(gi))
    return gi, gd, gy


def _query(rng, n_off=9, db=40, n=10):
    idx = np.full((n_off, 10), -1, np.int32)
    dist = np.full((n_off, 10), 1e300)
    shift = np.zeros((n_off, 10), np.int32)
    nc = np.full(n_off, min(n, db), np.int32)
    for o in range(n_off):
        k = nc[o]
        idx[o, :k] = rng.choice(db, k, replace=False)
        dist[o, :k] = rng.uniform(0.05, 0.6, k)
        shift[o, :k] = rng.integers(0, 60, k)
    return idx, dist, shift, nc


def test_merge_matches_oracle_random():
    rng = np.random.default_rng(3)
    for _ in range(50):
        _check(*_query(rng, db=int(rng.integers(10, 60))))


def test_smaller_distance_wins_and_first_wins_a_tie():
    idx = np.full((3, 10), -1, np.int32); dist = np.full((3, 10), 1e300); sh = np.zeros((3, 10), np.int32)
    idx[0, :2] = [7, 2]; dist[0, :2] = [0.2, 0.25]; sh[0, :2] = [1, 2]
    idx[1, :2] = [7, 2]; dist[1, :2] = [0.1, 0.25]; sh[1, :2] = [3, 4]     # 7: smaller wins; 2: a tie keeps offset 0's
    idx[2, :1] = [2]; dist[2, :1] = [0.2500000001]; sh[2, :1] = [5]        # equal once cast to float: still offset 0's
    gi, gd, gy = _check(idx, dist, sh, np.array([2, 2, 1], np.int32))
    assert list(gi) == [2, 7]
    assert gy[0] == GO.shift_to_yaw(2) and gy[1] == GO.shift_to_yaw(3)
    assert gd[1] == np.float32(0.1)


def test_float_comparison_decides():
    """Two distances that differ in double but not in float: the float comparison sees a tie, the first stays."""
    a = 0.2
    b = np.nextafter(a, 0.0)            # smaller in double, same float
    assert np.float32(a) == np.float32(b) and b < a
    idx = np.full((2, 10), -1, np.int32); dist = np.full((2, 10), 1e300); sh = np.zeros((2, 10), np.int32)
    idx[0, 0], dist[0, 0], sh[0, 0] = 4, a, 10
    idx[1, 0], dist[1, 0], sh[1, 0] = 4, b, 20
    _, _, gy = _check(idx, dist, sh, np.array([1, 1], np.int32))
    assert gy[0] == GO.shift_to_yaw(10)


def test_threshold_is_strict():
    idx = np.full((1, 10), -1, np.int32); dist = np.full((1, 10), 1e300); sh = np.zeros((1, 10), np.int32)
    idx[0, :3] = [1, 2, 3]; dist[0, :3] = [0.30, np.nextafter(0.30, 0.0), 0.31]
    gi, _, _ = _check(idx, dist, sh, np.array([3], np.int32))
    assert list(gi) == [2]


def test_empty_and_small_database():
    idx = np.full((9, 10), -1, np.int32); dist = np.full((9, 10), 1e300); sh = np.zeros((9, 10), np.int32)
    gi, _, _ = _check(idx, dist, sh, np.zeros(9, np.int32))              # empty database: nothing
    assert gi.size == 0
    rng = np.random.default_rng(5)
    for db in (1, 2, 3, 7):                                               # fewer than 10 entries: min(10, db) candidates each
        q = _query(rng, db=db)
        gi, _, _ = _check(*q)
        assert set(gi) <= set(range(db))
