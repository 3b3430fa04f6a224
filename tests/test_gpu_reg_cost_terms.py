"""GPU: the scan matcher's NDT, GICP and VGICP cost evaluations term by term against the restatement in reg_cost_ref.py, fed
the device's own tables (covariances and voxel lines read back), and the correspondence / fitness gates at thresholds whose
square is not a float.

* Sums: each of the 28 outputs lies within gamma(m - 1) * sum |t| of the exact sum of the m restated terms (any order of
  double additions stays inside it).
* One-point sources: the evaluation is the point's terms summed in offset order into zeros, so it must equal the restatement
  bit for bit.  Here a wrong voxel, cofactor or weight cannot hide in a sum.
* Correspondences: GICP's target index per point, NDT / VGICP's found / not-found pattern per (offset, point).
* Gates: the reference compares a float squared distance with a double threshold (fast_gicp_impl.hpp:141
  `k_sq_dists[0] < corr_dist_threshold_ * corr_dist_threshold_`; getFitnessScore `nn_dists[0] <= max_range`).  A point is
  planted at the float squared distance where rounding the threshold to float first would decide the other way."""
import math
import os

import numpy as np
import pytest

import reg_cost_ref as RC

pytestmark = pytest.mark.gpu

EMU = bool(os.environ.get("LSDREG_EMU"))          # SIMT emulator build: small clouds
F32 = np.float32
RATIO = {}                                        # worst |S - fsum| / ((m - 1) u sum |t|) per matcher
EXACT = {}                                        # one-point evaluations that matched bit for bit


def _cloud(P):
    P = np.asarray(P, F32).reshape(-1, 3)
    return np.ascontiguousarray(np.concatenate([P, np.zeros((P.shape[0], 1), F32)], 1))


@pytest.fixture(scope="module")
def scene():
    """test_gpu_reg.py's scene: block map in a local frame (NDT: always at test_gpu_reg.py's 0.25 m spacing), a scan at a
    perturbed guess and at the true pose."""
    from lsdreg import synth
    m = synth.block_map(1, 1, 1, 0.5 if EMU else 0.25)
    m[:, :2] -= np.array([60, 40], F32)
    dense = synth.block_map(1, 1, 1, 0.25)                             # NDT: voxels of more than 6 points (cheap to build)
    dense[:, :2] -= np.array([60, 40], F32)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = np.array([1.0, -2.0, 1.8])
    scan = synth.scan64(2, 60 if EMU else 200, Rgt, tgt + np.array([60, 40, 0]))[::2].copy()
    dR, dt = synth.perturb(5, 0.5, 3.0)
    guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
    Tgt = np.eye(4); Tgt[:3, :3] = Rgt; Tgt[:3, 3] = tgt
    T2 = Tgt.copy(); T2[:3, 3] += [0.03, -0.02, 0.01]
    return dict(tgt=m, dense=dense, src=scan, guess=guess, Tgt=Tgt, T2=T2)


def _sums(kind, dev, terms, deriv=True):
    e, H, b, nc = dev
    assert nc == terms.n_corr
    r = RC.check_sums(RC.unpack(e, H, b), terms.flat(), deriv)
    RATIO[kind] = max(RATIO.get(kind, 0.0), r)
    print(f"{kind}: m = {terms.flat().shape[0]}, worst |S - fsum| / ((m - 1) u sum|t|) = {r:.3g}; so far {RATIO}")


def _one_point(kind, dev, terms):
    """A one-point source's evaluation against the restated terms summed in offset order: bit for bit."""
    e, H, b, nc = dev
    assert nc == terms.n_corr
    got, want = RC.unpack(e, H, b), terms.per_point()[0]
    assert np.array_equal(got, want), (kind, np.nonzero(got != want)[0], got[got != want], want[got != want])
    EXACT[kind] = EXACT.get(kind, 0) + 1


def _pattern(g, terms):
    n_off, n = terms.found.shape
    corr = g.correspondences().reshape(n_off, n)
    assert np.array_equal(corr >= 0, terms.found), np.argwhere((corr >= 0) != terms.found)[:10]


# ------------------------------------------------------------------ NDT
@pytest.mark.parametrize("n_off", [1, 7, 27])
def test_ndt_terms(scene, n_off):
    import lsdreg
    src = scene["src"]
    g = lsdreg.Matcher("NDT_CUDA", ndt_neighbors=n_off)
    g.set_target(scene["dense"]); g.set_source(src)
    tab = RC.Table(g.voxels())
    for T in (scene["guess"], scene["Tgt"]):
        t = RC.ndt_terms(src, tab, 1.0, n_off, T, T)
        dev = g.cost(T)
        _pattern(g, t)
        assert t.used.sum() > (200 if EMU else 1000)
        _sums("ndt", dev, t)
    for deriv in (True, False):           # looked up at Tgt (the last linearisation), evaluated at T2
        t = RC.ndt_terms(src, tab, 1.0, n_off, scene["Tgt"], scene["T2"], deriv)
        _sums("ndt", g.cost(scene["T2"], update=False, deriv=deriv), t, deriv)
        _pattern(g, t)
    g.close()


@pytest.mark.parametrize("n_off", [1, 7, 27])
def test_ndt_one_point_sources(scene, n_off):
    """Planted one-point sources: scan points, points that the linearisation pose puts exactly on voxel faces (x / res - 0.5
    an integer in fp32), points in a 7-point and a 6-point voxel, a point with no voxel; linearised at T1, then evaluated at
    T2 with the correspondences of T1, with and without derivatives."""
    import lsdreg
    rng = np.random.default_rng(3)
    a7 = rng.uniform(0.55, 1.45, (7, 3)) + [2.0, 0.0, 50.0]          # voxel (2, 0, 50) of 7 points
    b6 = rng.uniform(0.55, 1.45, (6, 3)) + [-5.0, 0.0, 50.0]         # voxel (-5, 0, 50) of 6 points
    tgt = np.concatenate([scene["dense"], _cloud(np.concatenate([a7, b6]))])
    g = lsdreg.Matcher("NDT_CUDA", ndt_neighbors=n_off)
    g.set_target(tgt)
    tab = RC.Table(g.voxels())
    T1 = np.eye(4); T1[:3, 3] = [0.25, -0.5, 0.125]                   # exact in fp32: a + t lands where planted
    T2 = T1.copy(); T2[:3, 3] += [0.0625, 0.03125, -0.046875]
    scan = scene["src"][:, :3].astype(np.float64)
    world = scan @ scene["Tgt"][:3, :3].T + scene["Tgt"][:3, 3]         # the scan where it lies in the map
    near = world[np.linalg.norm(scan, axis=1) < 12.0][::97][:8] - T1[:3, 3]
    face = world[::211][:8].copy()
    face[:4, 0] = np.round(face[:4, 0] - 0.5) + 0.5                  # x / 1 - 0.5 an integer once transformed by T1
    face[4:, 2] = np.round(face[4:, 2] - 0.5) + 0.5
    planted = np.concatenate([near, face - T1[:3, 3], a7[:2] + 0.05 - T1[:3, 3], b6[:1] + 0.05 - T1[:3, 3],
                              [[2.5, 0.3, 51.0] - T1[:3, 3]], [[0.0, 0.0, 90.0]]]).astype(F32)
    lt = np.stack(RC.xform_f(T1, planted), 1)
    on_face = np.any(lt - F32(0.5) == np.round(lt - F32(0.5)), axis=1)
    assert on_face.sum() >= 8                                          # the faces are hit exactly in fp32
    hits = 0
    for p in planted:
        src = _cloud(p)
        g.set_source(src)
        t1 = RC.ndt_terms(src, tab, 1.0, n_off, T1, T1)
        _one_point("ndt", g.cost(T1), t1)
        hits += t1.used.any()
        for deriv in (True, False):
            _one_point("ndt", g.cost(T2, update=False, deriv=deriv), RC.ndt_terms(src, tab, 1.0, n_off, T1, T2, deriv))
    assert hits >= 10
    print(f"one-point sources matched bit for bit: {EXACT}")
    g.close()


# ------------------------------------------------------------------ GICP
@pytest.fixture(scope="module")
def thread_src(scene):
    """test_gicp_thread_shape_kernels_match_oracle's near-range scan: >= 16 384 points, the thread-per-point kernels."""
    from lsdreg import synth
    Tgt = scene["Tgt"]
    src = synth.scan64(3, 900, Tgt[:3, :3], Tgt[:3, 3] + np.array([60, 40, 0]))
    src = np.ascontiguousarray(src[np.linalg.norm(src[:, :3], axis=1) < 20.0])
    assert src.shape[0] >= 16384
    return src


def _gicp_case(g, src, tgt, poses, T2):
    tn, sn = g.covariances(True), g.covariances(False)
    for T in poses:
        corr, _ = RC.gicp_nn(src, tgt, T, 2.0)
        dev = g.cost(T)
        np.testing.assert_array_equal(g.correspondences(), corr)
        _sums("gicp", dev, RC.gicp_terms(src, tgt, sn, tn, corr, T, T))
    for deriv in (True, False):           # Mahalanobis matrices of the last linearisation (poses[-1]), evaluated at T2
        _sums("gicp", g.cost(T2, update=False, deriv=deriv), RC.gicp_terms(src, tgt, sn, tn, corr, poses[-1], T2, deriv), deriv)
        np.testing.assert_array_equal(g.correspondences(), corr)


@pytest.mark.parametrize("shape", ["warp", "thread"])
def test_gicp_terms(scene, thread_src, shape):
    import lsdreg
    src = scene["src"] if shape == "warp" else thread_src
    assert (src.shape[0] < 16384) == (shape == "warp")
    g = lsdreg.Matcher("FAST_GICP")
    g.set_target(scene["tgt"]); g.set_source(src)
    _gicp_case(g, src, scene["tgt"], (scene["guess"], scene["Tgt"]), scene["T2"])
    g.close()


def test_gicp_one_point_sources(scene):
    """One-point sources: the Mahalanobis matrix of the point's own (read back) normal and its target's, linearised at Tgt,
    then evaluated at T2 with that matrix."""
    import lsdreg
    g = lsdreg.Matcher("FAST_GICP")
    g.set_target(scene["tgt"])
    tn = g.covariances(True)
    T1, T2 = scene["Tgt"], scene["T2"]
    for p in scene["src"][::151][:24]:
        src = _cloud(p[:3])
        g.set_source(src)
        sn = g.covariances(False)
        corr, _ = RC.gicp_nn(src, scene["tgt"], T1, 2.0)
        _one_point("gicp", g.cost(T1), RC.gicp_terms(src, scene["tgt"], sn, tn, corr, T1, T1))
        for deriv in (True, False):
            _one_point("gicp", g.cost(T2, update=False, deriv=deriv), RC.gicp_terms(src, scene["tgt"], sn, tn, corr, T1, T2, deriv))
    print(f"one-point sources matched bit for bit: {EXACT}")
    g.close()


# ------------------------------------------------------------------ VGICP
def _vgicp_case(g, src, poses, T2, n_off):
    sn = g.covariances(False)
    tab = RC.Table(g.voxels())
    for T in poses:
        t = RC.vgicp_terms(src, sn, tab, 1.0, n_off, T, T)
        dev = g.cost(T)
        _pattern(g, t)
        _sums("vgicp", dev, t)
    for deriv in (True, False):
        t = RC.vgicp_terms(src, sn, tab, 1.0, n_off, poses[-1], T2, deriv)
        _sums("vgicp", g.cost(T2, update=False, deriv=deriv), t, deriv)
    return tab


@pytest.mark.parametrize("n_off", [1, 7, 27])
def test_vgicp_terms(scene, n_off):
    import lsdreg
    g = lsdreg.Matcher("FAST_VGICP", ndt_neighbors=n_off)
    g.set_target(scene["tgt"]); g.set_source(scene["src"])
    _vgicp_case(g, scene["src"], (scene["guess"], scene["Tgt"]), scene["T2"], n_off)
    g.close()


@pytest.fixture(scope="module")
def vg_edges():
    """A target of crowded voxels (test_gpu_reg_build.py's overfull map voxel: 1 000 points in one 0.4 m box) next to
    single-point voxels (a sparse line, 3 m apart), and sources around both and on floor(x / res - 0.5) boundaries."""
    rng = np.random.default_rng(5)
    crowd = rng.uniform(-0.2, 0.2, (1000, 3)) * [1.0, 1.0, 0.05] + [1.0, 1.0, 0.0]
    patch = np.concatenate([rng.uniform(-3, 3, (300, 2)), rng.normal(-1.5, 0.01, (300, 1))], 1)
    line = np.stack([np.arange(12) * 3.0 + 10.3, np.full(12, -7.7), np.full(12, 0.6)], 1)
    tgt = _cloud(np.concatenate([crowd, patch, line]))
    s_crowd = crowd[::50] + rng.normal(0, 0.05, (20, 3))
    s_patch = patch[::15] + rng.normal(0, 0.05, (20, 3))
    s_line = line + rng.normal(0, 0.2, line.shape)
    bound = np.concatenate([s_patch[:10], s_line[:6]])
    bound[:, 0] = np.round(bound[:, 0] - 0.5) + 0.5                    # x / 1 - 0.5 an integer in double
    bound[::2, 1] = np.round(bound[::2, 1] - 0.5) + 0.5
    src = _cloud(np.concatenate([s_crowd, s_patch, s_line, bound]))
    return dict(tgt=tgt, src=src, n_bound=len(bound))


@pytest.mark.parametrize("n_off", [1, 7, 27])
def test_vgicp_edges(vg_edges, n_off):
    import lsdreg
    g = lsdreg.Matcher("FAST_VGICP", ndt_neighbors=n_off)
    g.set_target(vg_edges["tgt"]); g.set_source(vg_edges["src"])
    counts = g.voxels()["count"]
    assert counts.max() >= 500 and (counts == 1).sum() >= 10           # crowded and single-point voxels both present
    I = np.eye(4)
    T2 = np.eye(4); T2[:3, 3] = [0.02, -0.01, 0.015]
    tab = _vgicp_case(g, vg_edges["src"], (T2, I), T2, n_off)         # linearised last at the identity: boundaries exact
    t = RC.vgicp_terms(vg_edges["src"], g.covariances(False), tab, 1.0, n_off, I, I)
    assert t.used.sum() > 40
    # one-point sources: the point's own normal (read back), every voxel it reaches
    for p in vg_edges["src"][::3]:
        src = _cloud(p[:3])
        g.set_source(src)
        sn = g.covariances(False)
        _one_point("vgicp", g.cost(I), RC.vgicp_terms(src, sn, tab, 1.0, n_off, I, I))
        for deriv in (True, False):
            _one_point("vgicp", g.cost(T2, update=False, deriv=deriv), RC.vgicp_terms(src, sn, tab, 1.0, n_off, I, T2, deriv))
    print(f"one-point sources matched bit for bit: {EXACT}")
    g.close()


def test_vgicp_one_point_sources(scene):
    import lsdreg
    g = lsdreg.Matcher("FAST_VGICP", ndt_neighbors=7)
    g.set_target(scene["tgt"])
    tab = RC.Table(g.voxels())
    T1, T2 = scene["Tgt"], scene["T2"]
    for p in scene["src"][::151][:24]:
        src = _cloud(p[:3])
        g.set_source(src)
        sn = g.covariances(False)
        _one_point("vgicp", g.cost(T1), RC.vgicp_terms(src, sn, tab, 1.0, 7, T1, T1))
        for deriv in (True, False):
            _one_point("vgicp", g.cost(T2, update=False, deriv=deriv), RC.vgicp_terms(src, sn, tab, 1.0, 7, T1, T2, deriv))
    print(f"one-point sources matched bit for bit: {EXACT}")
    g.close()


# ------------------------------------------------------------------ gates
def _f32_sq(x):
    x = F32(x)
    return F32(x * x)


def _edge_below(D):
    """A float offset x on one axis whose fp32 squared length is the largest plantable float below D^2 (double), as the
    reference's gate `(double) d2 < D * D` admits it.  Returns (d2, (x, 0))."""
    G = float(D) * float(D)
    x0 = F32(math.sqrt(G))
    best = None
    for k in range(-64, 65):
        x = F32(x0 + F32(k) * np.spacing(x0))
        d2 = _f32_sq(x)
        if float(d2) < G and (best is None or d2 > best[0]):
            best = (d2, (x, F32(0)))
    return best


def _edge_two_axes(lo, G):
    """(x, y) with lo < fp32 d2 < G (double), for a threshold no single axis reaches."""
    x0 = F32(math.sqrt(G))
    for i in range(0, 200):
        x = F32(x0 - F32(i) * np.spacing(x0))
        for j in range(1, 4000):
            y = F32(j) * F32(2.0 ** -20)
            d2 = F32(_f32_sq(x) + _f32_sq(y))
            if float(d2) >= G:
                break
            if d2 > lo:
                return d2, (x, y)
    return None


def _gate_plant(D):
    """The planted offsets of a correspondence-gate case: the largest plantable d2 below D^2 (accepted by the reference),
    and d2 = f32(D)^2 (accepted by the reference unless D^2 is exact).  For thresholds whose fp32 search bound
    f32(f32(D)^2) falls below a plantable d2 < D^2, that d2 instead (on two axes if no single axis reaches it)."""
    G = float(D) * float(D)
    old_bound = _f32_sq(D)
    below = _edge_below(D)
    if below[0] <= old_bound:                      # nothing between f32(D)^2 and D^2 on one axis: try two
        two = _edge_two_axes(old_bound, G)
        if two is not None:
            below = two
    at = (old_bound, (F32(D), F32(0)))
    return below, at, G


@pytest.mark.parametrize("D", [0.7, 0.9, 0.137, 0.5, 2.0, 5.0, 25.0])
@pytest.mark.parametrize("shape", ["warp", "thread"])
def test_corr_gate(D, shape):
    """Source points at the origin and at z = 100 (identity pose: the fp32 transform is exact), each with one target point
    at a planted offset.  Correspondences must be those of the reference's gate (float d2 against double D^2) and of the
    oracle; the thread shape pads the source to 16 384 points with a grid 500 m away."""
    import lsdreg
    from oracle.reg import OracleMatcher
    (d_b, (xb, yb)), (d_a, (xa, ya)), G = _gate_plant(D)
    if D == 0.137:
        assert float(d_b) < G and d_b > _f32_sq(D)             # a point the old fp32 search bound lost
    tgt = _cloud([[xb, yb, 0.0], [xa, ya, 100.0]])
    src = [[0.0, 0.0, 0.0], [0.0, 0.0, 100.0]]
    if shape == "thread":
        gx, gy = np.meshgrid(np.arange(128.0), np.arange(128.0))
        src = np.concatenate([src, np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, -500.0)], 1)])
    src = _cloud(src)
    I = np.eye(4)
    corr, d2 = RC.gicp_nn(src, tgt, I, D)
    assert corr[0] == 0 and d2[0] == d_b and d2[1] == d_a        # the planted distances, as the kernels compute them
    assert corr[1] == (1 if float(d_a) < G else -1) and (corr[2:] == -1).all()
    g = lsdreg.Matcher("FAST_GICP", max_corr_dist=D)
    g.set_target(tgt); g.set_source(src)
    dev = g.cost(I)
    np.testing.assert_array_equal(g.correspondences(), corr)
    _sums("gicp", dev, RC.gicp_terms(src, tgt, g.covariances(False), g.covariances(True), corr, I, I))
    g.close()
    o = OracleMatcher("gicp", max_corr=D)
    o.set_target(tgt); o.set_source(src)
    o.cost(I)
    np.testing.assert_array_equal(o.corr, corr)


def _fitness_plant(r):
    """An offset whose fp32 d2 is f32(r) when f32(r) > r (a point the reference does not count and an fp32 gate would),
    else the largest fp32 d2 <= r (counted by both)."""
    r32 = F32(r)
    x0 = F32(math.sqrt(r))
    cands = []
    for k in range(-64, 65):
        x = F32(x0 + F32(k) * np.spacing(x0))
        cands.append((_f32_sq(x), x))
    if float(r32) > r:
        hit = [c for c in cands if c[0] == r32]
        assert hit, "no single-axis offset reaches f32(max_range)"
        return hit[0]
    return max(c for c in cands if float(c[0]) <= r)


@pytest.mark.parametrize("max_range", [0.3, 0.6, 0.5, 2.0, 5.0, 25.0])
@pytest.mark.parametrize("shape", ["warp", "thread"])
def test_fitness_gate(max_range, shape):
    """getFitnessScore(max_range) with a source point at the planted distance and one at 0.25 m (always counted): the
    score and count of the reference's gate (float d2 <= double max_range), through Matcher.fitness, LoopDetector.fitness
    and the oracle."""
    import lsdreg
    from oracle.reg import OracleMatcher
    d_p, x = _fitness_plant(max_range)
    tgt = _cloud([[x, 0.0, 0.0], [0.25, 0.0, 100.0]])
    src = [[0.0, 0.0, 0.0], [0.0, 0.0, 100.0]]
    if shape == "thread":
        gx, gy = np.meshgrid(np.arange(128.0), np.arange(128.0))
        src = np.concatenate([src, np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, -500.0)], 1)])
    src = _cloud(src)
    d2 = [float(d_p), 0.0625]
    kept = [v for v in d2 if v <= max_range]
    want = math.fsum(kept) / len(kept)
    I = np.eye(4)
    g = lsdreg.Matcher("FAST_GICP")
    g.set_target(tgt); g.set_source(src)
    assert g.fitness(max_range, T=I) == want
    g.close()
    d = lsdreg.LoopDetector()
    a = d.add_keyframe(tgt, 0.0); b = d.add_keyframe(src, 0.0)
    score, n = d.fitness(a, b, I.astype(F32), max_range)
    # calc_fitness_score: points with nothing within the grid search radius get their exact neighbour (500 m away)
    assert n == len(kept) and score == want
    d.close()
    o = OracleMatcher("gicp")
    o.set_target(tgt); o.set_source(src)
    assert o.fitness(T=I, max_range=max_range) == want
