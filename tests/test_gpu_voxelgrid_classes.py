"""GPU: the voxel grid's leaf classes, bit for bit against the restated pcl::VoxelGrid (oracle.oracle.voxelgrid).
A leaf of up to SMALL points is summed by one thread after a sorting network; a crowded leaf (up to CAP points) by one warp after
a bitonic sort of its members in shared memory; a big leaf by one block, sorted in the block's shared memory (up to BIG points)
or in place in global memory (above BIG)."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SMALL, CAP, BIG = 8, 512, 4096     # kVgSmall, kVgCap, kVgBig in csrc/voxelgrid.cu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _leaf(rng, k, cell, leaf=0.5):
    p = np.empty((k, 4), np.float32)
    p[:, :3] = np.asarray(cell, np.float64) * leaf + rng.uniform(0.01, 0.49, (k, 3)) * (leaf / 0.5)
    p[:, 3] = 10.0 ** rng.uniform(-2, 3, k)     # five orders of magnitude: any change of summation order shows
    return p


def _exact(vg, pts, leaf=0.5):
    from oracle import oracle as O
    want = O.voxelgrid(pts[np.isfinite(pts[:, :3]).all(1)], leaf)     # non-finite points are skipped
    got = vg.filter(np.ascontiguousarray(pts), leaf)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    return got


@pytest.fixture(scope="module")
def vg():
    import lsdreg
    lsdreg.init(0)
    g = lsdreg.VoxelGrid(max_points=200000)
    yield g
    g.close()


@pytest.mark.parametrize("order", ["blocks", "reverse", "shuffled", "interleaved"])
def test_class_boundaries(vg, order):
    rng = np.random.default_rng(3)
    sizes = (1, SMALL - 1, SMALL, SMALL + 1, 31, 32, 33, CAP - 1, CAP, CAP + 1)
    parts = [_leaf(rng, k, (4 * j, -3 * j, j % 4)) for j, k in enumerate(sizes)]
    bg = _leaf(rng, 20000, (0, 0, 0))
    bg[:, :3] = rng.uniform(-30, 30, (20000, 3)) * [1, 1, 0.2]
    pts = np.concatenate(parts + [bg])
    if order == "reverse":
        pts = pts[::-1]
    elif order == "shuffled":
        pts = pts[rng.permutation(pts.shape[0])]
    elif order == "interleaved":     # crowded leaves' members alternate with each other and with the background in input order
        key = np.concatenate([np.arange(p.shape[0]) / p.shape[0] for p in parts + [bg]])
        pts = pts[np.argsort(key, kind="stable")]
    _exact(vg, pts)


@pytest.mark.parametrize("k", [2473, BIG, BIG + 1, 5000])
def test_big_leaves(vg, k):
    rng = np.random.default_rng(k)
    big = _leaf(rng, k, (2, 1, 0))
    pts = np.concatenate([big, _leaf(rng, 3, (9, 9, 0)), _leaf(rng, 600, (-4, 0, 1))])
    _exact(vg, pts[rng.permutation(pts.shape[0])])
    _exact(vg, big)     # every point in one leaf


def test_more_crowded_leaves_than_warps_in_flight(vg):
    rng = np.random.default_rng(5)
    cells = np.stack(np.meshgrid(np.arange(60), np.arange(60), np.arange(2), indexing="ij"), -1).reshape(-1, 3)   # 7200 leaves
    k = rng.integers(SMALL + 1, 40, cells.shape[0])
    pts = np.concatenate([_leaf(rng, int(kk), c) for kk, c in zip(k, cells)])
    _exact(vg, pts[rng.permutation(pts.shape[0])][:200000])


def test_non_finite_points_inside_crowded_leaves(vg):
    rng = np.random.default_rng(6)
    a, b = _leaf(rng, 100, (1, 1, 1)), _leaf(rng, 700, (3, 1, 1))
    a[[5, 50, 99], [0, 1, 2]] = [np.nan, np.inf, -np.inf]
    b[[0, 300, 699], [2, 0, 1]] = [np.inf, np.nan, np.nan]
    pts = np.concatenate([a, b, _leaf(rng, 9, (0, 4, 0)), _leaf(rng, 2, (5, 5, 0))])
    _exact(vg, pts[rng.permutation(pts.shape[0])])


def test_back_to_back_calls_with_different_grids(vg):
    """Scratch comes back idle: a second call on another grid gives what a fresh handle gives."""
    import lsdreg
    rng = np.random.default_rng(8)
    first = np.concatenate([_leaf(rng, 600, (0, 0, 0)), _leaf(rng, 12, (50, 3, 1))])
    second = np.concatenate([_leaf(rng, 40, (-7, 2, 0), 0.2), _leaf(rng, 5, (100, -40, 3), 0.2)])
    _exact(vg, first)
    got = _exact(vg, second, 0.2)
    fresh = lsdreg.VoxelGrid(max_points=1000)
    assert np.array_equal(fresh.filter(second, 0.2).view(np.uint32), got.view(np.uint32))
    fresh.close()
    _exact(vg, first)


def test_bench_scans(vg):
    sys.path.insert(0, ROOT)
    import bench
    for s in range(23):
        _exact(vg, np.asarray(bench.make_step(s)[0], np.float32))
