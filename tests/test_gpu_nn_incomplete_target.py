"""GPU: nearest-neighbour searches against a target whose point map could not hold every point, and fitness scores whose
nearest neighbours lie past the 64-voxel grid search.

The matcher indexes its target in a hash-voxel point map and uses it as an exact nearest-neighbour index for GICP
correspondences (gicp_corr_kernel / gicp_corr_thread_kernel) and for getFitnessScore (fitness_range: Matcher.fitness, the
loop detector's coarse fitness and calc_fitness_score, the global aligner's fitness).  The map refuses a point of a voxel
that already holds 896 points, of a full probe chain, or beyond +-2^18 voxels, and which points of an overfull voxel it
refuses depends on the order of the insert's atomics.  Every consumer is compared here with a brute-force reference:

* correspondences and fp32 d2: reg_cost_ref.gicp_nn (the kernels' fp32 transform and dist2, ties to the lower index);
* cost sums: reg_cost_ref.gicp_terms within gamma(m - 1) sum |t| of the exact sum (check_sums);
* fitness: fsum of the brute-force d2 <= max_range over their count; the count exact, the score within (m - 1) u sum |t|.

Scenes: a plane patch plus one box of V points centred on a voxel centre (V = 896 is the last complete voxel, 897 the
first incomplete one; every box point is also a source point, so at the identity its nearest neighbour is itself at
d2 = 0 and every refused point shows up as a wrong correspondence); a 2^12-line table with one target point per voxel;
target points beyond +-2^18 voxels; nearest neighbours at 20, 31.9, 32.1, 45 and 90 m with max_range from exactly the
cap (1024 m^2 at 0.5 m) to DBL_MAX.  Each runs in both kernel shapes: below and at or above 16 384 source points.

On the device the set of refused points changes from build to build, so fresh handles on the overfull target must give
the same bits, and the loop detector's decisions on a key frame with such a voxel must be those of the restatement."""
import math
import os

import numpy as np
import pytest

import reg_cost_ref as RC

pytestmark = pytest.mark.gpu

EMU = bool(os.environ.get("LSDREG_EMU"))          # SIMT emulator build: small scenes, warp shape only
F32 = np.float32
DBL_MAX = 1.7976931348623157e308
SHAPES = ["warp"] if EMU else ["warp", "thread"]
CAP = 64.0 * 0.5 * 0.5 * 64.0                     # fitness_search_sq's cap at the default 0.5 m map resolution


def _cloud(P):
    P = np.asarray(P, F32).reshape(-1, 3)
    return np.ascontiguousarray(np.concatenate([P, np.zeros((P.shape[0], 1), F32)], 1))


def _pad(src, shape, z=-500.0):
    """test_corr_gate's padding: the thread shape gets a 128 x 128 grid 500 m below everything (no correspondence)."""
    if shape == "warp":
        assert src.shape[0] < 16384
        return src
    gx, gy = np.meshgrid(np.arange(128.0), np.arange(128.0))
    out = np.concatenate([src, _cloud(np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, z)], 1))])
    assert out.shape[0] >= 16384
    return out


def _plane(rng):
    """A 6 m x 6 m patch at z = -1.5 (a few points per voxel) around the box."""
    g = np.arange(-2.0, 4.0, 0.23)
    gx, gy = np.meshgrid(g, g)
    P = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, -1.5)], 1)
    return P + rng.uniform(-0.02, 0.02, P.shape)


def overfull_scene(V, shape):
    """Plane patch plus a box of V distinct points in (1, 1, 0) +- 0.18: voxel (2, 2, 0) at 0.5 m (pos2grid rounds, so it
    is centred on (1, 1, 0)) holds all of them.  Source: every box point, points 0.3 m around the box, every 5th plane point."""
    rng = np.random.default_rng(V)
    box = np.unique(rng.uniform(-0.18, 0.18, (V + 64, 3)).astype(F32), axis=0)[:V]
    box = rng.permutation(box) + F32(1.0)
    box[:, 2] -= F32(1.0)
    assert len(box) == V and np.all(np.round(box / F32(0.5)) == [2, 2, 0])
    plane = _plane(rng)
    tgt = _cloud(np.concatenate([plane, box]))
    around = np.array([1.0, 1.0, 0.0]) + rng.uniform(-0.5, 0.5, (64, 3))
    src = _pad(_cloud(np.concatenate([box, around, plane[::5]])), shape)
    return src, tgt, len(plane)


def full_table_scene(shape):
    """One target point per voxel in a 2^12-line table (EMU: 2^10): more voxels than lines, so the probe chains fill.
    Source: every 3rd target point moved by 1 cm, whose nearest neighbour is that point."""
    nx, ny, nz = (20, 20, 15) if not EMU else (12, 12, 10)
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3) * 0.5
    rng = np.random.default_rng(7)
    tgt = _cloud(g + rng.uniform(-0.1, 0.1, g.shape) + [-3.0, -3.0, -2.0])
    src = tgt[::3].copy()
    src[:, :3] += F32(0.01)
    return _pad(src, shape), tgt, (12 if not EMU else 10)


def far_coord_scene(shape):
    """A cluster near the origin and one beyond +-2^18 voxels (|x| > 131 072 m at 0.5 m); source points 0.1 m from
    points of both."""
    rng = np.random.default_rng(11)
    near = rng.uniform(-2.0, 2.0, (300, 3))
    far = np.array([140000.0, -50.0, 3.0]) + rng.uniform(-2.0, 2.0, (300, 3))
    farx = np.array([-1.0, 200000.0, 0.0]) + rng.uniform(-2.0, 2.0, (100, 3))
    tgt = _cloud(np.concatenate([near, far, farx]))
    P = tgt[:, :3].astype(np.float64)
    src = _cloud(np.concatenate([P[::7] + [0.1, 0.0, 0.0], P[300::5] + [0.0, 0.1, 0.0]]))
    return _pad(src, shape), tgt


FAR = np.array([20.0, 31.9, 32.1, 45.0, 90.0])


def far_nn_scene(shape):
    """Target points 400 m apart, each with one source point straight above it at a distance of FAR; the thread shape
    pads with points within 0.5 m of the first target point (found at once by the grid search)."""
    P = np.stack([np.arange(len(FAR)) * 400.0, np.zeros(len(FAR)), np.zeros(len(FAR))], 1)
    tgt = _cloud(np.concatenate([P, P + [0.3, 0.0, 0.0]]))
    src = P + np.stack([np.zeros(len(FAR)), np.zeros(len(FAR)), FAR], 1)
    if shape == "thread":
        gx, gy = np.meshgrid(np.arange(128.0), np.arange(128.0))
        src = np.concatenate([src, np.stack([gx.ravel() / 256.0, gy.ravel() / 256.0, np.full(gx.size, 0.25)], 1)])
    return _cloud(src), tgt


# ------------------------------------------------------------------ references
def want_fitness(d2, max_range):
    """(exact mean, count, bound): fsum of the fp32 d2 <= max_range (compared in double) over their count m, and how far
    the device's mean may lie from it: the (m - 1) u sum |t| any order of m double additions may miss the sum by, over m,
    plus the rounding of the division (and of the exact mean itself)."""
    kept = d2.astype(np.float64)[d2.astype(np.float64) <= max_range]
    if kept.size == 0:
        return DBL_MAX, 0, 0.0
    s = math.fsum(kept)
    w = s / kept.size
    return w, kept.size, (max(kept.size - 1, 0) * RC.U64 * s / kept.size + 2 * RC.U64 * w) * (1 + 1e-9)


def check_fitness(got, d2, max_range, n_got=None):
    w, n, bnd = want_fitness(d2, max_range)
    if n_got is not None:
        assert n_got == n, (n_got, n)
    if n == 0:
        assert got == DBL_MAX
    else:
        assert abs(got - w) <= bnd, (got, w, got - w, bnd)


def nn(src, tgt, T, max_corr=2.0):
    return RC.gicp_nn(src, tgt, T, max_corr)


# ------------------------------------------------------------------ consumers
def check_matcher(src, tgt, poses, max_ranges, **kw):
    """Matcher("FAST_GICP"): cost(T) then correspondences() at each pose, the cost sums, fitness(max_range, T)."""
    import lsdreg
    g = lsdreg.Matcher("FAST_GICP", **kw)
    g.set_target(tgt); g.set_source(src)
    tn, sn = g.covariances(True), g.covariances(False)
    for T in poses:
        corr, d2 = nn(src, tgt, T)
        e, H, b, nc = g.cost(T)
        got = g.correspondences()
        bad = np.nonzero(got != corr)[0]
        assert bad.size == 0, f"{bad.size} of {int((corr >= 0).sum())} correspondences wrong, first {bad[:8]}"
        terms = RC.gicp_terms(src, tgt, sn, tn, corr, T, T)
        assert nc == terms.n_corr
        RC.check_sums(RC.unpack(e, H, b), terms.flat())
        for mr in max_ranges:
            check_fitness(g.fitness(mr, T=T), d2, mr)
    g.close()


def check_loop(src, tgt, T, max_ranges):
    """LoopDetector with the cloud as the target slot: fitness() (score and count) at T, and the fitness column of
    match() (getFitnessScore(fitness_score_max_range) at the candidate's final pose)."""
    import lsdreg
    for mr in max_ranges:
        d = lsdreg.LoopDetector(fitness_score_max_range=mr)
        a = d.add_keyframe(tgt, 0.0); b = d.add_keyframe(src, 0.0)
        score, n = d.fitness(a, b, T.astype(F32), mr)
        check_fitness(score, nn(src, tgt, T.astype(F32).astype(np.float64))[1], mr, n)
        m = d.match(a, [b], T[None])
        Tf = m["final"][0]
        check_fitness(m["fitness"][0], nn(src, tgt, Tf)[1], mr)
        d.close()


def check_galign(src, tgt, T, max_ranges):
    """GlobalAligner with the cloud as the reference slot: the fitness of match() at the pair's final pose, batched and
    serial the same bits."""
    import lsdreg
    for mr in max_ranges:
        ga = lsdreg.GlobalAligner(fitness_score_max_range=mr)
        r = ga.add_keyframe(tgt, True); s = ga.add_keyframe(src, False)
        m = ga.match(s, [r], T[None])
        check_fitness(m["fitness"][0], nn(src, tgt, m["final"][0])[1], mr)
        ms = ga.match(s, [r], T[None], serial=True)
        assert np.array_equal(ms["final"], m["final"]) and np.array_equal(ms["fitness"], m["fitness"])
        ga.close()


def _poses():
    I = np.eye(4)
    T1 = I.copy(); T1[:3, 3] = [0.0625, -0.03125, 0.015625]
    from lsdreg import synth
    T2 = I.copy(); T2[:3, :3] = synth.rot_from_rpy(0.002, -0.001, 0.01); T2[:3, 3] = [0.02, 0.01, -0.01]
    return I, T1, T2


OVERFULL_V = [896, 897] if EMU else [896, 897, 1500, 3000]


@pytest.mark.parametrize("V", OVERFULL_V)
@pytest.mark.parametrize("shape", SHAPES)
def test_overfull_voxel(V, shape):
    src, tgt, n_plane = overfull_scene(V, shape)
    I, T1, T2 = _poses()
    corr, d2 = nn(src, tgt, I)
    assert np.array_equal(corr[:V], np.arange(n_plane, len(tgt))) and not d2[:V].any()   # each box point's own match
    check_matcher(src, tgt, (I, T1, T2), (0.01, 25.0, DBL_MAX))
    check_loop(src, tgt, I, (25.0, DBL_MAX))
    check_galign(src, tgt, I, (25.0, 1e4))


@pytest.mark.parametrize("shape", SHAPES)
def test_full_table(shape):
    src, tgt, l2 = full_table_scene(shape)
    import lsdreg
    m = lsdreg.HashVoxelMap(0.5, l2)
    m.insert(tgt)
    assert m.stats()["dropped"] > 0, "the table must refuse points"
    m.close()
    I, T1, _ = _poses()
    check_matcher(src, tgt, (I, T1), (25.0, DBL_MAX), map_log2_lines=l2)


@pytest.mark.parametrize("shape", SHAPES)
def test_out_of_range_coordinates(shape):
    src, tgt = far_coord_scene(shape)
    I, T1, _ = _poses()
    corr, _ = nn(src, tgt, I)
    assert (corr[43:][:100] >= 300).all()                      # source points beside the far clusters have their match
    check_matcher(src, tgt, (I, T1), (25.0, DBL_MAX))
    check_loop(src, tgt, I, (25.0, DBL_MAX))
    check_galign(src, tgt, I, (25.0,))


@pytest.mark.skipif(EMU, reason="grid searches out to 64 voxels take minutes on the emulator")
@pytest.mark.parametrize("shape", SHAPES)
def test_fitness_past_the_grid_search(shape):
    """getFitnessScore(max_range) with max_range at the 64-voxel cap and past it: every consumer counts the neighbours
    beyond 32 m that PCL counts."""
    src, tgt = far_nn_scene(shape)
    I = np.eye(4)
    _, d2 = nn(src, tgt, I)
    np.testing.assert_allclose(np.sqrt(d2[:len(FAR)].astype(np.float64)), FAR, rtol=1e-6)
    mrs = (CAP, 1e4, DBL_MAX)
    check_matcher(src, tgt, (I,), mrs)
    check_loop(src, tgt, I, mrs)
    check_galign(src, tgt, I, mrs)
    from oracle.reg import OracleMatcher
    o = OracleMatcher("gicp")
    o.set_target(tgt); o.set_source(src)
    for mr in mrs:
        check_fitness(o.fitness(T=I, max_range=mr), d2, mr)


@pytest.mark.skipif(EMU, reason="the emulator inserts in order; the spread between builds is a device property")
def test_overfull_target_is_reproducible():
    """Four fresh matchers on the 3000-point voxel: the same align pose, iteration log and fitness, bit for bit."""
    import lsdreg
    src, tgt, _ = overfull_scene(3000, "warp")
    guess = np.eye(4, dtype=F32); guess[:3, 3] = [0.08, -0.05, 0.03]
    runs = []
    for _ in range(4):
        g = lsdreg.Matcher("FAST_GICP")
        g.set_target(tgt); g.set_source(src)
        out = g.align(guess)
        runs.append((out, g.final()[0], g.iteration_log(), g.fitness(25.0), g.fitness(DBL_MAX)))
        g.close()
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert np.array_equal(a, b)


def test_ref_matcher_fitness_on_overfull_voxel():
    """The compiled reference's getFitnessScore (k-d tree, no map) on the 1500-point voxel, at the identity."""
    from oracle import oracle as O
    if not O.HAVE_REF_REG:
        pytest.skip("oracle/_ref/libref_reg.so not built")
    import lsdreg
    from oracle.reg import RefMatcher
    src, tgt, _ = overfull_scene(897 if EMU else 1500, "warp")
    _, d2 = nn(src, tgt, np.eye(4))
    r = RefMatcher("gicp")
    r.set_target(tgt); r.set_source(src)
    g = lsdreg.Matcher("FAST_GICP")
    g.set_target(tgt); g.set_source(src)
    for mr in (0.01, 25.0, DBL_MAX):
        ref = r.fitness(mr)
        check_fitness(ref, d2, mr)
        check_fitness(g.fitness(mr, T=np.eye(4)), d2, mr)
    g.close()


# ------------------------------------------------------------------ loop closure next to a wall
RADIUS, STEP, N_KF = 10.0, 3.0, 22


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _blob_world():
    """test_gpu_loop.py's circle of key frames; the new key frame (the last) also sees a dense blob of 3000 points in one
    voxel 1 m from its sensor, as a wall next to the sensor gives."""
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    est, clouds, accum = [], [], []
    L = 2 * np.pi * RADIUS
    for i in range(N_KF):
        s = min(i * STEP, L)
        th = s / RADIUS
        R = synth.rot_from_rpy(0.0, 0.0, th + np.pi / 2)
        t = c0 + np.array([RADIUS * np.cos(th), RADIUS * np.sin(th), 0.0])
        f = s / L
        est.append(_pose(synth.rot_from_rpy(0.0, 0.0, np.deg2rad(5.0) * f) @ R, t + np.array([0.7, 0.7, 0.0]) * f))
        clouds.append(synth.scan64(100 + i, (200, 250, 400)[i % 3], R, t))
        accum.append(s)
    rng = np.random.default_rng(5)
    blob = rng.uniform(-0.2, 0.2, (3000, 3)) + [1.0, 0.0, 0.0]
    clouds[-1] = np.concatenate([clouds[-1], _cloud(blob)[:, :clouds[-1].shape[1]]]).astype(F32)
    return np.array(est), clouds, np.array(accum)


@pytest.mark.skipif(EMU, reason="the emulator inserts in order; the spread between builds is a device property")
def test_loop_detect_next_to_a_wall_is_reproducible():
    """Three fresh detectors give the same detect() bits (relpose, scores, information) on a new key frame with a
    3000-point voxel, and the decisions of the restatement (tests/loop_oracle.py)."""
    import lsdreg
    import loop_oracle as LO
    est, clouds, accum = _blob_world()
    new, kfs = [N_KF - 1], list(range(N_KF - 2))
    outs = []
    for _ in range(3):
        d = lsdreg.LoopDetector()
        for c, a in zip(clouds, accum):
            d.add_keyframe(c, a)
        outs.append((d.detect(est, kfs, new), d.reports()))
        d.close()
    for loops, reps in outs[1:]:
        assert reps == outs[0][1]
        assert len(loops) == len(outs[0][0])
        for a, b in zip(loops, outs[0][0]):
            for k in ("key1", "key2", "relpose", "coarse_score", "score", "information"):
                assert np.array_equal(a[k], b[k]), k
    loops, reps = outs[0]
    o = LO.OracleLoopDetector(clouds, accum)
    oloops, oreps = o.detect(est, kfs, new)
    names = ["skipped", "no_candidates", "coarse_reject", "gicp_diverged", "gicp_reject", "found"]
    assert [names[r["decision"]] for r in reps] == [r["decision"] for r in oreps]
    assert len(loops) == len(oloops)
    for g, ol in zip(loops, oloops):
        assert (g["key1"], g["key2"]) == (ol["key1"], ol["key2"])
        np.testing.assert_allclose(g["score"], ol["score"], rtol=1e-5)
        np.testing.assert_allclose(g["information"], ol["information"], rtol=1e-6)
