"""TEST INFRASTRUCTURE: the voxel grid's two leaf classes at their boundaries, run by tests/test_emu_voxelgrid_classes.py against
the SIMT emulator build.  A leaf of up to 8 points is summed by one thread (sorting network), one of up to 512 by a warp (bitonic
sort in shared memory), a larger one by a block (sorted in the block's shared memory up to 4096 points, in global memory above).  Every bit of every centroid must equal the restated
pcl::VoxelGrid's (sequential fp32 sums in input order)."""
import sys

import numpy as np

import lsdreg
from oracle import oracle as O

lsdreg.init(0)
rng = np.random.default_rng(7)
SMALL, CAP = 8, 512


def leaf_points(k, cell):
    """k points inside the 0.5 m leaf `cell`, channels spanning orders of magnitude so that any change of order shows."""
    c = np.asarray(cell, np.float64) * 0.5
    p = np.empty((k, 4), np.float32)
    p[:, :3] = c + rng.uniform(0.01, 0.49, (k, 3))
    p[:, 3] = 10.0 ** rng.uniform(-2, 3, k)
    return p


def check(vg, pts, name):
    got = vg.filter(pts, 0.5)
    want = O.voxelgrid(pts[np.isfinite(pts[:, :3]).all(1)], 0.5)   # non-finite points are skipped
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), name
    print("ok", name, want.shape[0])
    sys.stdout.flush()


vg = lsdreg.VoxelGrid(max_points=8000, log2_max_cells=20)
sizes = (1, SMALL - 1, SMALL, SMALL + 1, 31, 32, 33, CAP, CAP + 1)
parts = [leaf_points(k, (3 * j, -2 * j, j % 3)) for j, k in enumerate(sizes)]
background = leaf_points(1500, (0, 0, 0))
background[:, :3] = rng.uniform(-20, 20, (1500, 3)) * [1, 1, 0.2]
mixed = np.concatenate(parts + [background])
check(vg, np.ascontiguousarray(mixed), "class boundaries, leaves in blocks")
check(vg, np.ascontiguousarray(mixed[::-1]), "class boundaries, reverse input order")
check(vg, np.ascontiguousarray(mixed[rng.permutation(mixed.shape[0])]), "class boundaries, shuffled")
check(vg, leaf_points(3000, (1, 1, 1)), "one leaf of 3000 points (a block's)")
check(vg, np.concatenate([leaf_points(4500, (1, 1, 1)), leaf_points(40, (0, 3, 0))])[::-1].copy(), "a leaf of 4500 points (sorted in global memory)")
nan_leaf = leaf_points(40, (2, 2, 0))
nan_leaf[[3, 17, 29], 0] = [np.nan, np.inf, -np.inf]
check(vg, np.concatenate([nan_leaf, leaf_points(9, (4, 0, 0))]), "non-finite points inside a crowded leaf")
check(vg, leaf_points(20, (0, 5, 0)), "a second grid on the same handle")
print("FUZZ_VG_CLASSES_OK")
