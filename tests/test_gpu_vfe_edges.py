"""GPU parity of the detection voxelizer (lsd_vfe_*) at its edges, against the sequential numpy restatement
(oracle/vfe.py) and, where it is built, the compiled reference (oracle/_ref/libref_vfe.so).

Edges: a window at the max_points cap (the returned totals reach max_points + max_frame_num - 1) and empty realtime
frames; NaN and +-inf coordinates in the newest and in older, motion-compensated frames; points on the range faces and
one ulp either side, on grids whose extent is not a whole number of voxels; num_feature 4 / 5 / 8 x max_points_per_voxel
1 / 3 / 5 in both coordinate orders and both id modes; fp16 rounding ties, subnormals and overflow; a window of 1.2 M
points (two trips of the scan's carry loop); and the grid-size limit of lsd_vfe_create.

Bars: the same totals, voxel count, order, index rows and point counts as the oracle (per voxel key in unordered-id
mode); fp16 features bit for bit against the oracle fed the device's own window (any NaN equals any NaN); the window
itself bit for bit (the oracle rounds the transform's fma chain exactly)."""
import os

import numpy as np
import pytest

import vfe_edges as E

pytestmark = pytest.mark.gpu

HAVE_REF = os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_vfe.so"))
needs_ref = pytest.mark.skipif(not HAVE_REF or bool(os.environ.get("LSDREG_EMU")),
                               reason="oracle/_ref/libref_vfe.so not built (needs the reference tree + nvcc), or no device to run it")



def _pair(**kw):
    """A device voxelizer and the oracle with the same parameters."""
    import lsdreg
    from oracle.vfe import OracleVoxelizer
    g = lsdreg.Voxelizer(**kw)
    p = g.params
    o = OracleVoxelizer(min_range=tuple(p.min_range), max_range=tuple(p.max_range), voxel_size=tuple(p.voxel_size),
                        max_ppv=p.max_points_per_voxel, max_voxels=p.max_voxels, max_points=p.max_points, nf=p.num_feature,
                        max_frames=p.max_frame_num)
    return g, o


def _same_bits(a, b):
    """Element-wise bit equality of two float arrays, any NaN equal to any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    u = np.uint16 if a.dtype == np.float16 else np.uint32
    return (a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))


def _assert_same_bits(a, b, what):
    eq = _same_bits(a, b)
    if not eq.all():
        bad = np.argwhere(~eq)[:5]
        raise AssertionError(f"{what}: {int((~eq).sum())} elements differ, first at {bad.tolist()}: "
                             f"{[(a[tuple(i)], b[tuple(i)]) for i in bad]}")


def _key(idx, zyx=True):
    """Voxel key (x, y, z) of index rows."""
    x, y, z = (idx[:, 3], idx[:, 2], idx[:, 1]) if zyx else (idx[:, 1], idx[:, 2], idx[:, 3])
    return (z.astype(np.int64) << 42) | (y.astype(np.int64) << 21) | x.astype(np.int64)


def _check_window(g, o):
    win = g.points()
    assert win.shape == (o.total, g.params.num_feature)
    _assert_same_bits(win, o.buf[:o.total], "window")
    return win


def _check_voxels(g, o, win, zyx=True):
    """The device's voxelization of its window against the oracle on the same window; returns the device's rows."""
    feat, idx, npts = g.voxelize(zyx)
    of, oi, on = o.voxelize(points=win, zyx=zyx)
    assert feat.shape == of.shape
    if g.params.unordered_ids:
        kg, ko = np.argsort(_key(idx, zyx)), np.argsort(_key(oi, zyx))
        feat, idx, npts, of, oi, on = feat[kg], idx[kg], npts[kg], of[ko], oi[ko], on[ko]
        assert len(np.unique(_key(idx, zyx))) == idx.shape[0]
    np.testing.assert_array_equal(idx, oi)
    np.testing.assert_array_equal(npts, on)
    _assert_same_bits(feat, of, "fp16 features")
    return feat, idx, npts


# ------------------------------------------------------------------------------------------------------------- window cap
@pytest.mark.parametrize("max_points", [100, 1000])
@pytest.mark.parametrize("frames", [1, 2, 3, 4])
def test_window_at_the_max_points_cap(max_points, frames):
    """Streams of frames at, below and above max_points with empty frames mixed in.  The totals follow the reference's
    arithmetic, which reaches max_points + max_frame_num - 1 rows; the window and its voxelization match the oracle after
    every frame; an empty frame's row is the far row, never read from the caller; realtime=False empties the window."""
    from oracle.vfe import FAR_ROW_XYZ
    rng = np.random.default_rng(7 * max_points + frames)
    M = max_points
    g, o = _pair(max_points=M, max_frame_num=frames, max_voxels=100000)
    sizes = [M, M, M, M, 0, M // 2, 3 * M, 0, 0, 1, M - 1, M, 2, 0, M, M, M, M]
    peak = 0
    for step, n in enumerate(sizes):
        pts = E.cloud(rng, n, 5)
        pts[:, 4] = 0.01 * step
        mot = E.motion(rng)
        tg = g.accumulate(pts, mot)
        to = o.accumulate(pts, mot)
        assert tg == to, (step, tg, to)
        assert 1 <= tg <= M + frames - 1
        peak = max(peak, tg)
        win = _check_window(g, o)
        if n == 0:
            np.testing.assert_array_equal(win[0, :3], np.float32(FAR_ROW_XYZ))
            np.testing.assert_array_equal(win[0, 3:], 0.0)
        _check_voxels(g, o, win, zyx=bool(step % 2))
    assert peak == M + frames - 1                                   # the bound is reached, so the buffers are exercised
    # realtime=False: a fresh window of at most max_points rows, then a realtime frame on top of it
    for n in (M + 7, 0, 3):
        pts = E.cloud(rng, n, 5)
        assert g.accumulate(pts, None, realtime=False) == o.accumulate(pts, None, realtime=False) == min(n, M)
        _check_voxels(g, o, _check_window(g, o))
        mot = E.motion(rng)
        pts = E.cloud(rng, M, 5)
        assert g.accumulate(pts, mot) == o.accumulate(pts, mot)
        _check_voxels(g, o, _check_window(g, o))


def test_empty_realtime_frame_reads_nothing_from_the_caller():
    """num_points = 0 with a NULL point pointer: the library writes the one counted row itself; with realtime = 0 the
    window is empty."""
    import ctypes as C
    import lsdreg
    from oracle.vfe import FAR_ROW_XYZ
    g = lsdreg.Voxelizer(max_points=1000, max_frame_num=2)
    m = np.eye(4, dtype=np.float32)
    tot = C.c_int()
    lsdreg.capi.check(lsdreg.lib.lsd_vfe_accumulate(g.h, None, 0, m.ctypes.data, 1, C.byref(tot)))
    assert tot.value == 1
    w = g.points()
    np.testing.assert_array_equal(w, np.array([[FAR_ROW_XYZ] * 3 + [0, 0]], np.float32))
    feat, idx, npts = g.voxelize()
    assert feat.shape[0] == 0
    lsdreg.capi.check(lsdreg.lib.lsd_vfe_accumulate(g.h, None, 0, None, 0, C.byref(tot)))
    assert tot.value == 0 and g.points().shape == (0, 5) and g.voxelize()[0].shape[0] == 0


# ------------------------------------------------------------------------------------------------------------ non-finite
@pytest.mark.parametrize("nf", [5, 8])
def test_nonfinite_points_in_new_and_old_frames(nf):
    """NaN on an axis lands in cell 0 of that axis, and a NaN point of an older frame is NaN on all three.  +-inf is out
    of range; in an older frame it stays infinite on one axis while the transform makes others NaN (0 * inf under a
    yaw-only motion).  Window and voxels bit for bit against the oracle, after every frame."""
    rng = np.random.default_rng(11 + nf)
    g, o = _pair(num_feature=nf, max_frame_num=3)
    saw_nan_cell = 0
    for f, pts in enumerate(E.nonfinite_frames(rng, nf)):
        mot = E.motion(rng, yaw_only=f == 1)
        assert g.accumulate(pts, mot) == o.accumulate(pts, mot)
        win = _check_window(g, o)
        feat, idx, npts = _check_voxels(g, o, win)
        nanrow = np.isnan(feat[:, :3].astype(np.float32)).any(1)
        saw_nan_cell += int(nanrow.sum())
        assert (idx[nanrow][:, 1:] == 0).any(1).all()               # a NaN coordinate sits in cell 0 of some axis
    assert saw_nan_cell >= 15


# ------------------------------------------------------------------------------------------------------------------ faces
@pytest.mark.parametrize("grid", list(E.GRIDS))
@pytest.mark.parametrize("zyx", [True, False])
def test_range_faces(grid, zyx):
    """Bit for bit against the oracle at the faces: min is in, max is out, whatever the cell arithmetic says."""
    gp = E.GRIDS[grid]
    pts = E.face_points(gp)
    g, o = _pair(**gp)
    assert g.accumulate(pts, None, realtime=False) == o.accumulate(pts, None, realtime=False) == pts.shape[0]
    win = _check_window(g, o)
    feat, idx, npts = _check_voxels(g, o, win, zyx)
    assert 0 < feat.shape[0] < pts.shape[0]
    ijk, in_range, in_grid = o.cells(pts)
    mx = np.asarray(gp["max_range"], np.float32)
    on_max = pts[:, :3] == mx
    for a in range(3):     # rounded up: on every axis, some max-face point lies inside a grid cell
        assert ((on_max[:, a] & in_grid).sum() >= 2) == (grid == "odd_up")
    if grid == "odd_down":  # rounded down: some points in range lie in the cut last cell
        assert (in_range & ~in_grid).sum() >= 6
    assert not (in_range & in_grid)[on_max.any(1)].any()


# ----------------------------------------------------------------------------------------------------------------- shapes
@pytest.mark.parametrize("nf", [4, 5, 8])
@pytest.mark.parametrize("ppv", [1, 3, 5])
@pytest.mark.parametrize("zyx", [True, False])
@pytest.mark.parametrize("unordered", [0, 1])
def test_shapes(nf, ppv, zyx, unordered):
    """Three motion-compensated frames of clustered points (voxels of 1 to ~12 points) at every shape; the window carries
    every feature past z and adds 0.1 to the time channel only when there is one."""
    rng = np.random.default_rng(100 * nf + 10 * ppv + 2 * zyx + unordered)
    g, o = _pair(num_feature=nf, max_points_per_voxel=ppv, max_frame_num=3, max_points=20000, unordered_ids=unordered)
    for f in range(3):
        pts = E.cloud(rng, 3000, nf)
        mot = E.motion(rng)
        assert g.accumulate(pts, mot) == o.accumulate(pts, mot)
        win = _check_window(g, o)
        feat, idx, npts = _check_voxels(g, o, win, zyx)
        assert npts.max() == ppv and ((npts < ppv).any() or ppv == 1)
        if f:
            old = win[pts.shape[0]:]
            prev = o_prev[:old.shape[0]]
            np.testing.assert_array_equal(old[:, 3], prev[:, 3])
            if nf > 4:
                np.testing.assert_array_equal(old[:, 4], (prev[:, 4].astype(np.float64) + 0.1).astype(np.float32))
                np.testing.assert_array_equal(old[:, 5:], prev[:, 5:])
        o_prev = win.copy()


# ------------------------------------------------------------------------------------------------------------------- fp16
@pytest.mark.parametrize("nf", [5, 8])
def test_fp16_rounding_of_features(nf):
    """One-point voxels hold the value itself: its fp16 bits must be numpy's astype(float16).  Voxels of 2 to 5 points hold
    fp32 means of such values: bit for bit against the oracle."""
    rng = np.random.default_rng(5 + nf)
    v = E.fp16_values(rng)
    n = v.shape[0]
    rows = []
    for k in range(1, 6):                                   # n voxels of k points: x cell j, y cell per k
        q = np.zeros((n * k, nf), np.float32)
        q[:, 0] = np.repeat(np.float32(-59.95) + np.float32(0.1) * np.arange(n, dtype=np.float32), k)
        q[:, 1] = np.float32(10.05 + 2 * k)
        q[:, 2] = np.float32(0.5)
        for f in range(3, nf):
            q[:, f] = v[(np.arange(n * k) * (2 * k - 1) + 7 * f) % n] if k > 1 else np.roll(v, f)
        rows.append(q)
    pts = np.concatenate(rows)
    g, o = _pair(num_feature=nf, max_points=pts.shape[0])
    assert g.accumulate(pts, None, realtime=False) == o.accumulate(pts, None, realtime=False) == pts.shape[0]
    feat, idx, npts = _check_voxels(g, o, _check_window(g, o))
    one = npts == 1
    assert one.sum() == n and feat.shape[0] == 5 * n
    with np.errstate(over="ignore"):
        want = rows[0][:, 3:].astype(np.float16)
    _assert_same_bits(feat[one][:, 3:], want, "one-point voxel features against astype(float16)")
    wf = want.astype(np.float32)
    assert ((np.abs(wf) < 6.1e-5) & (wf != 0)).sum() >= 5 and np.isinf(wf).sum() >= 6


# ------------------------------------------------------------------------------------------------------------------ scale
def test_scale_two_carry_trips():
    """1.2 M points (1172 scan blocks: the carry loop of vfe_scan_kernel runs twice); voxelize twice, identical."""
    rng = np.random.default_rng(3)
    g, o = _pair(max_points=1_200_000, max_frame_num=2, max_voxels=2_000_000)
    for f in range(2):
        p = np.zeros((600_000, 5), np.float32)
        p[:, :3] = rng.uniform((-63.9, -63.9, -1.9), (63.9, 63.9, 3.9), (600_000, 3))
        p[:300_000:3, :3] = p[1:300_001:3, :3] + np.float32(0.01)                         # shared voxels
        p[:, 3] = rng.uniform(0, 255, 600_000)
        mot = E.motion(rng)
        assert g.accumulate(p, mot) == o.accumulate(p, mot) == 600_000 * (f + 1)
    win = _check_window(g, o)
    feat, idx, npts = _check_voxels(g, o, win)
    assert feat.shape[0] > 1_048_576 // 2
    f2, i2, n2 = g.voxelize(True)
    np.testing.assert_array_equal(i2, idx)
    np.testing.assert_array_equal(n2, npts)
    np.testing.assert_array_equal(f2.view(np.uint16), feat.view(np.uint16))


# -------------------------------------------------------------------------------------------------------- create limits
def test_create_rejects_grids_whose_keys_overflow():
    """Voxel keys (z * gs1 + y) * gs0 + x are 32-bit: gs0 * gs1 * gs2 must stay below 2^31.  Just under the limit the
    last cell still voxelizes."""
    import lsdreg
    with pytest.raises(lsdreg.LsdError):
        lsdreg.Voxelizer(voxel_size=(0.001, 0.001, 0.15))
    with pytest.raises(lsdreg.LsdError):
        lsdreg.Voxelizer(min_range=(0, 0, 0), max_range=(1024, 1024, 2048), voxel_size=(1, 1, 1), max_points=100)
    gp = dict(min_range=(0, 0, 0), max_range=(1024, 1024, 2047), voxel_size=(1, 1, 1), max_points=100)
    g, o = _pair(**gp)
    p = np.array([[1023.5, 1023.5, 2046.5, 1, 0], [0.5, 0.5, 0.5, 2, 0], [1023.5, 0.5, 2046.5, 3, 0]], np.float32)
    g.accumulate(p, None, realtime=False); o.accumulate(p, None, realtime=False)
    feat, idx, npts = _check_voxels(g, o, _check_window(g, o))
    np.testing.assert_array_equal(idx[0], [0, 2046, 1023, 1023])


# ---------------------------------------------------------------------------------------------- the compiled reference
def _ref_rows(r, zyx=True):
    """The compiled reference's output split into rows that hold points and rows that hold none (all features NaN: a
    key its hash pass inserted for a point its voxelization pass then rejects at a range face)."""
    rf, ri = r.voxelize(zyx)
    empty = np.isnan(rf.astype(np.float32)).all(1)
    return rf[~empty], ri[~empty], int(empty.sum())


def _against_ref(g, o, r, win, zyx=True):
    """Per voxel key: the device's voxel set equals the reference's; features bit for bit where every point of the voxel
    is in the mean and the sum has one order (one point), within 1 fp16 ulp where several are summed in another order."""
    feat, idx, npts = g.voxelize(zyx)
    rf, ri, n_empty = _ref_rows(r, zyx)
    ijk, in_range, in_grid = o.cells(win)
    real = in_range & in_grid
    phantom = in_grid & ~in_range
    keys = lambda c: (c[:, 2] << 42) | (c[:, 1] << 21) | c[:, 0]
    n_phantom = len(np.setdiff1d(np.unique(keys(ijk[phantom])), np.unique(keys(ijk[real]))))
    assert n_empty == n_phantom
    kg, kr = np.argsort(_key(idx, zyx)), np.argsort(_key(ri, zyx))
    np.testing.assert_array_equal(idx[kg], ri[kr])
    raw = np.unique(keys(ijk[real]), return_counts=True)
    raw_cnt = dict(zip(raw[0].tolist(), raw[1].tolist()))
    kk = _key(idx[kg], zyx)
    full = np.array([raw_cnt[int(k)] <= g.params.max_points_per_voxel for k in kk])
    single = np.array([raw_cnt[int(k)] == 1 for k in kk])
    a, b = feat[kg], rf[kr]
    _assert_same_bits(a[single], b[single], "one-point voxels against the compiled reference")
    a32, b32 = a[full].astype(np.float32), b[full].astype(np.float32)
    np.testing.assert_allclose(a32, b32, rtol=1e-3, atol=1e-7)
    return n_phantom


@needs_ref
@pytest.mark.parametrize("nf", [5, 8])
def test_nonfinite_against_compiled_reference(nf):
    """NaN on an axis: the compiled reference also puts the point in cell 0 of that axis; its window has the same bits."""
    from oracle.vfe import RefVoxelizer
    rng = np.random.default_rng(11 + nf)
    g, o = _pair(num_feature=nf, max_frame_num=3)
    r = RefVoxelizer(num_feature=nf, max_frame_num=3)
    frames = E.nonfinite_frames(rng, nf)
    for f, pts in enumerate(frames[:1] if nf != 5 else frames):   # num_feature != 5: the reference's window transform
        mot = E.motion(rng, yaw_only=f == 1)                       # copies features 3 and 4 only; one frame there
        assert g.accumulate(pts, mot) == o.accumulate(pts, mot) == r.accumulate(pts, mot)
        win = g.points()
        _assert_same_bits(win, r.points(), "window against the compiled reference")
        assert _against_ref(g, o, r, win) == 0


@needs_ref
@pytest.mark.parametrize("grid", list(E.GRIDS))
def test_range_faces_against_compiled_reference(grid):
    """The same voxels as the compiled reference at the faces.  Where the grid size rounds up, the reference also emits a
    row of NaN features for each max-face cell that only its range test rejects (its hash pass has no range test); the
    product emits none."""
    from oracle.vfe import RefVoxelizer
    gp = E.GRIDS[grid]
    pts = E.face_points(gp)
    g, o = _pair(**gp)
    r = RefVoxelizer(**gp)
    g.accumulate(pts, None, realtime=False); o.accumulate(pts, None, realtime=False); r.accumulate(pts, None, realtime=False)
    n_phantom = _against_ref(g, o, r, g.points())
    assert (n_phantom > 0) == (grid == "odd_up")


@needs_ref
@pytest.mark.parametrize("nf", [4, 5, 8])
@pytest.mark.parametrize("ppv", [1, 3, 5])
@pytest.mark.parametrize("zyx", [True, False])
def test_shapes_against_compiled_reference(nf, ppv, zyx):
    """One frame at every shape: the same voxel set as the compiled reference, the same features where it is deterministic."""
    from oracle.vfe import RefVoxelizer
    rng = np.random.default_rng(100 * nf + 10 * ppv + 2 * zyx)
    g, o = _pair(num_feature=nf, max_points_per_voxel=ppv, max_points=20000)
    r = RefVoxelizer(num_feature=nf, max_points_per_voxel=ppv, max_points=20000)
    pts = E.cloud(rng, 3000, nf)
    g.accumulate(pts, None, realtime=False); o.accumulate(pts, None, realtime=False); r.accumulate(pts, None, realtime=False)
    _against_ref(g, o, r, g.points(), zyx)
