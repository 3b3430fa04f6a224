"""Edge sets of the detection voxelizer, shared by tests/test_gpu_vfe_edges.py (device against the oracle and the compiled
reference) and tests/test_vfe_oracle_host.py (the oracle against a per-point restatement, on the CPU)."""
import numpy as np

DEFAULT = dict(min_range=(-64.0, -64.0, -2.0), max_range=(64.0, 64.0, 4.0), voxel_size=(0.1, 0.1, 0.15))
# Grids whose extent is not a whole number of voxels, with negative minimums.  (max - min) / vs = 21.6, 25.9, 14.7: the grid
# size rounds up on every axis, so a point on a max face lies in a grid cell and only the range test rejects it.
# 21.3, 25.3, 14.3: it rounds down, so points in range but in the cut last cell are rejected by the grid test alone.
ODD_UP = dict(min_range=(-3.3, -7.05, -1.1), max_range=(5.35, 2.0, 3.3), voxel_size=(0.4, 0.35, 0.3))
ODD_DOWN = dict(min_range=(-3.3, -7.05, -1.1), max_range=(5.2, 1.8, 3.2), voxel_size=(0.4, 0.35, 0.3))
GRIDS = dict(default=DEFAULT, odd_up=ODD_UP, odd_down=ODD_DOWN)


def cloud(rng, n, nf, lo=(-6.0, -6.0, -1.5), hi=(6.0, 6.0, 2.5), clustered=0.5):
    """n points in a box, a share of them in tight clusters so that voxels hold more than 5 points."""
    p = np.zeros((n, nf), np.float32)
    p[:, :3] = rng.uniform(lo, hi, (n, 3))
    k = int(n * clustered)
    if k:
        centres = rng.uniform(lo, hi, (max(k // 12, 1), 3))
        p[:k, :3] = centres[rng.integers(0, centres.shape[0], k)] + rng.uniform(-0.03, 0.03, (k, 3))
        p[:n] = p[rng.permutation(n)]
    p[:, 3:] = rng.uniform(0.0, 255.0, (n, nf - 3))
    if nf > 4:
        p[:, 4] = 0.0
    return p


def motion(rng, yaw_only=False):
    """A small rigid motion; yaw_only leaves exact zeros in the matrix, so the transform meets 0 * inf."""
    r, p, y = rng.uniform(-0.02, 0.02, 3)
    if yaw_only:
        r = p = 0.0
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    M = np.eye(4, dtype=np.float32)
    M[:3, :3] = Rz @ Ry @ Rx
    M[:3, 3] = rng.uniform(-0.5, 0.5, 3)
    return M


def nonfinite_frames(rng, nf=5):
    """Three frames of the default range; the first two carry NaN / +-inf in x, y and z: on one axis with the others in
    range, next to a coordinate out of range, on all three axes, and in a feature.  A NaN coordinate puts its point in
    cell 0 of that axis, where no finite point of these frames lies."""
    frames = []
    for f in range(3):
        p = cloud(rng, 2000, nf, lo=(-20, -20, -1.5), hi=(20, 20, 3.0))
        p[:, 4 if nf > 4 else 3] = 0.5 * f
        if f < 2:
            rows = []
            for a in range(3):
                for v in (np.nan, np.inf, -np.inf):
                    for other in (0.0, 0.3, 100.0):                        # the next axis: in range twice, out once
                        r = np.array(([-30.0 - 3 * f, 40.0 + 2 * a, 0.2 + 0.4 * a, 7.0, 0.0] + [1.0] * 3)[:nf], np.float32)
                        r[(a + 1) % 3] += other
                        r[a] = v
                        rows.append(r)
            r = np.full(nf, np.nan, np.float32); r[3:] = 1.0; rows.append(r)      # NaN everywhere
            r = np.array(([-50.0, 50.0, np.nan, np.nan, 0.0] + [2.0] * 3)[:nf], np.float32); rows.append(r)  # NaN feature
            ins = rng.choice(p.shape[0], len(rows), replace=False)
            p[ins] = np.array(rows)
        frames.append(p)
    return frames


def face_points(grid, nf=5):
    """Points on the min and max faces of every axis and one ulp either side, on interior cell boundaries min + k*vs and
    one ulp either side, and on corners; the other coordinates at distinct cell centres."""
    mn, mx, vs = (np.asarray(grid[k], np.float32) for k in ("min_range", "max_range", "voxel_size"))
    gs = np.round((mx - mn) / vs).astype(int)
    up, dn = np.float32(np.inf), np.float32(-np.inf)
    rows = []
    j = 0
    for a in range(3):
        vals = []
        for face in (mn[a], mx[a]):
            vals += [np.nextafter(face, dn), face, np.nextafter(face, up)]
        for k in (1, 2, gs[a] // 2, gs[a] - 1, gs[a]):
            b = np.float32(mn[a] + np.float32(k) * vs[a])
            vals += [np.nextafter(b, dn), b, np.nextafter(b, up)]
        for v in vals:
            r = np.zeros(nf, np.float32)
            for b in range(3):
                c = (j * 3 + 2 * b + 1) % gs[b]
                r[b] = mn[b] + (np.float32(c) + np.float32(0.5)) * vs[b]
            r[a] = v
            r[3:] = np.float32(j % 251)
            rows.append(r)
            j += 1
    for cx in (0, 1):
        for cy in (0, 1):
            for cz in (0, 1):
                for d in (dn, None, up):
                    r = np.zeros(nf, np.float32)
                    for b, c in enumerate((cx, cy, cz)):
                        face = mx[b] if c else mn[b]
                        r[b] = face if d is None else np.nextafter(face, d)
                    r[3:] = np.float32(j % 251)
                    rows.append(r)
                    j += 1
    return np.array(rows, np.float32)


def fp16_values(rng):
    """fp32 values whose fp16 rounding is delicate: ties between neighbouring halves (both parities, both signs),
    subnormals and values under half the smallest one, the overflow threshold 65520 and beyond, and infinities."""
    h = rng.integers(0x0400, 0x7bff, 200).astype(np.uint16).view(np.float16)          # normal halves, not the largest
    lo, hi = h.astype(np.float32), np.nextafter(h, np.float16(np.inf)).astype(np.float32)
    ties = (lo + hi) * np.float32(0.5)                                                    # exact in fp32
    sub = np.array([1e-6, -1e-6, 2.98e-8, 2.9802322e-08, 5.9604645e-08, 8.940697e-08, 3e-5, 6.097555e-05, 6.1035156e-05,
                    1.0000001e-6, 1.5e-6], np.float32)
    big = np.array([65504, 65519.996, 65520, 65536, 1e5, -1e5, 3.4e38, -65520, np.inf, -np.inf], np.float32)
    v = np.concatenate([ties, -ties, lo, sub, big, ties * np.float32(1.0000001)])
    return v.astype(np.float32)
