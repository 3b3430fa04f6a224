"""GPU parity: fused k-NN + plane + residual/Jacobian + reduction (K3-K5), the iterated ESKF update
and map_incremental, against the CPU oracle, through the C ABI.
Bars (BASELINE.json north_star): neighbour ids bit-exact; pose within 1e-4 m / 1e-5 rad."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POS_TOL, ROT_TOL = 1e-4, 1e-5


def _pair(small_world, reference_order=True, **kw):
    import lsdreg
    from oracle import eskf
    from oracle.lio import OracleLio
    m = small_world["map"]
    g = lsdreg.LioFrontend(map_log2_lines=20, **kw)
    g.set_reference_order(reference_order)        # on is the library's default
    g.map.insert(m, 0)
    g.set_next_id(m.shape[0])
    kw.pop("eskf_literal", None)
    # stale_neighbours=True: the reference's Nearest_Points rows outlive a search that finds nothing — the product's default
    o = OracleLio(kw.get("ivox_nearby", 18), knn_exact=bool(kw.get("knn_mode_exact", 0)), expected_cells=1 << 18, stale_neighbours=True,
                  reference_order=reference_order)
    o.add_map_points(m)
    prior = eskf.State()
    prior.rot = eskf.R_to_quat(small_world["Rprior"])
    prior.pos = small_world["tprior"].copy()
    return g, o, prior


def _rot_err(qa, qb):
    from oracle import eskf
    return np.linalg.norm(eskf.so3_log(eskf.quat_mul(eskf.quat_conj(qa), qb)))


@pytest.mark.parametrize("kw", [dict(), dict(ivox_nearby=74), dict(knn_mode_exact=1), dict(reference_order=False),
                                dict(reference_order=False, ivox_nearby=74)])
def test_linearize_matches_oracle(small_world, kw):
    """Nearest_Points rows in the order IVox::GetClosestPoint returns them (the default: libstdc++'s nth_element on the
    reference's candidate sequence) — ids compared position by position against the oracle, which is pinned id for id to the
    compiled iVox; the planes then carry the compiled esti_plane's bits.  kw reference_order=False: ascending (d2, id) rows."""
    from oracle import oracle as O
    g, o, prior = _pair(small_world, **kw)
    n = g.load_scan(small_world["scan"])
    body = g.get_down()
    ref_body = O.voxelgrid(small_world["scan"], 0.5)
    assert n == ref_body.shape[0]
    # feed the oracle the SAME downsampled cloud (SURVEY.md §7: K1 parity is tolerance-level)
    o.near_xyz = np.zeros((n, 5, 3), np.float32); o.near_ids = np.full((n, 5), -1, np.int32)
    o.near_cnt = np.zeros(n, np.int32); o.selected = np.ones(n, np.uint8)
    o.world = np.zeros((n, 4), np.float32); o.plane = np.zeros((n, 4), np.float32)
    ro = o._hmodel(body, prior, True)
    rg = g.linearize(prior.to_vec(), True)
    mt = g.get_matches()
    assert (mt["world"][:, :3].view(np.int32) == o.world[:, :3].view(np.int32)).all()
    assert (mt["cnt"] == o.near_cnt).all()
    assert (mt["idx"] == o.near_ids).all()                      # bit-exact neighbour indices
    assert (mt["selected"] == o.selected[:n]).all()
    sel = mt["selected"].astype(bool)
    assert (mt["plane"][sel].view(np.int32) == o.plane[sel].view(np.int32)).all()
    assert rg["n_eff"] == ro["n"] and rg["n_eff"] > 1000
    np.testing.assert_allclose(rg["HTH"], o.last["HTH6"], rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(rg["HTh"], o.last["HTh6"], rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(rg["res_sum"], o.last["res_sum"], rtol=1e-12)
    # second evaluation without search reuses neighbours and the selected flags
    st2 = prior.copy(); st2.pos = st2.pos + np.array([0.01, -0.02, 0.005])
    ro2 = o._hmodel(body, st2, False)
    rg2 = g.linearize(st2.to_vec(), False)
    assert rg2["n_eff"] == ro2["n"]
    np.testing.assert_allclose(rg2["HTH"], o.last["HTH6"], rtol=1e-10, atol=1e-9)


@pytest.mark.parametrize("literal,ref_order", [(1, True), (0, True), (0, False)])
def test_update_pose_parity_and_map_incremental(small_world, literal, ref_order):
    from oracle import eskf
    g, o, prior = _pair(small_world, reference_order=ref_order, eskf_literal=literal)
    n = g.load_scan(small_world["scan"])
    body = g.get_down()
    P0 = eskf.init_P()
    r = o.process_scan(body, prior, P0, downsample=False, update_map=False)
    xg, Pg, info = g.update(prior.to_vec(), P0)
    xo = o.x.to_vec()
    assert info["iterations"] == r["iters"]
    assert np.abs(xg[0:3] - xo[0:3]).max() < POS_TOL
    assert _rot_err(xg[3:7], xo[3:7]) < ROT_TOL
    np.testing.assert_allclose(xg, xo, atol=1e-7)
    np.testing.assert_allclose(Pg, o.P, rtol=1e-4, atol=1e-12)  # literal and Schur forms both
    # converged onto the ground truth (scan noise 2 cm)
    assert np.abs(xg[0:3] - small_world["tgt"]).max() < 0.02
    # map_incremental: same add / skip decision for every point, same resulting map
    added_o = o.map_incremental(body)
    added_g = g.map_incremental(xo)  # same state on both sides
    flags, _ = g.get_map_flags()
    bad = np.nonzero(flags != o.flags)[0]
    assert not len(bad), f"map_incremental flags differ at {bad[:8]}: {flags[bad[:8]]} vs {o.flags[bad[:8]]}"
    assert added_g == added_o
    st = g.map.stats()
    assert st["points"] == o.map.num_points and st["cells"] == o.map.num_cells


def test_scan_sequence_full_pipeline(small_world):
    """Three consecutive scans through lsd_lio_scan (host pointers): pose parity at every step."""
    import lsdreg
    from lsdreg import synth
    from oracle import eskf
    g, o, prior = _pair(small_world)
    x = prior.to_vec(); P = eskf.init_P()
    xo_state = prior.copy(); Po = P.copy()
    for k in range(3):
        Rk = small_world["Rgt"] @ synth.rot_from_rpy(0, 0, 0.02 * k)
        tk = small_world["tgt"] + np.array([0.4 * k, 0.1 * k, 0.0])
        scan = synth.scan64(10 + k, 250, Rk, tk)
        # prior = previous posterior + inflated covariance (stands in for IMU propagation noise)
        P = P + np.eye(23) * 1e-2
        Po = Po + np.eye(23) * 1e-2
        x, P, info = g.scan(scan, x, P)
        assert info["status"] == lsdreg.OK and info["n_eff"] > 1000
        # oracle consumes the GPU's downsampled cloud so k-NN inputs are identical
        r = o.process_scan(g.get_down(), xo_state, Po, downsample=False)
        xo_state, Po = o.x.copy(), o.P.copy()
        xo = xo_state.to_vec()
        assert np.abs(x[0:3] - xo[0:3]).max() < POS_TOL, k
        assert _rot_err(x[3:7], xo[3:7]) < ROT_TOL, k
        assert abs(info["n_added"] - r["added"]) <= 3, k
        assert np.abs(x[0:3] - tk).max() < 0.05


def test_first_scan_seeds_map_and_small_scan_is_skipped(small_world):
    import lsdreg
    from oracle import eskf
    g = lsdreg.LioFrontend(map_log2_lines=18)
    x = lsdreg.make_state(pos=small_world["tgt"], rot_xyzw=eskf.R_to_quat(small_world["Rgt"]))
    P = lsdreg.init_cov()
    x1, P1, info = g.scan(small_world["scan"], x, P)
    assert info["status"] == lsdreg.MAP_SEEDED
    assert g.map.stats()["points"] == info["n_down"] == info["n_added"]
    np.testing.assert_array_equal(x1, x)
    tiny = small_world["scan"][:3].copy()
    x2, P2, info = g.scan(tiny, x, P)
    assert info["status"] == lsdreg.SCAN_TOO_SMALL
    np.testing.assert_array_equal(x2, x); np.testing.assert_array_equal(P2, P)


def test_no_effective_points(small_world):
    import lsdreg
    g = lsdreg.LioFrontend(map_log2_lines=18)
    g.map.insert(small_world["map"][:1000], 0)
    x = lsdreg.make_state(pos=(5000.0, 5000.0, 0.0))  # nowhere near the map
    P = lsdreg.init_cov()
    x1, P1, info = g.scan(small_world["scan"], x, P)
    assert info["status"] == lsdreg.NO_EFFECTIVE_POINTS and info["n_eff"] == 0
    np.testing.assert_array_equal(x1, x)


def test_prefetch_is_transparent(small_world):
    """Double-buffered ingest (lsd_lio_prefetch): poses are bit-identical to the serial path, whatever the caller
    prefetches — the right scan, a scan it then does not register, or two scans in a row."""
    import lsdreg
    from lsdreg import synth
    from oracle import eskf
    scans = []
    for k in range(4):
        Rk = small_world["Rgt"] @ synth.rot_from_rpy(0, 0, 0.02 * k)
        tk = small_world["tgt"] + np.array([0.4 * k, 0.1 * k, 0.0])
        scans.append(np.ascontiguousarray(synth.scan64(10 + k, 250, Rk, tk)))
    decoy = np.ascontiguousarray(scans[0][::-1] + np.float32(3.0))

    def run(mode):
        g, o, prior = _pair(small_world)
        x = prior.to_vec(); P = eskf.init_P()
        out = []
        if mode == "pipelined":
            g.prefetch(scans[0])
        for k in range(4):
            if mode == "pipelined" and k + 1 < 4:
                g.prefetch(scans[k + 1])
            if mode == "decoy":
                g.prefetch(decoy)                      # never registered: must not leak into scan k
                if k == 2:
                    g.prefetch(scans[3])               # two pending prefetches; the second one is used next round
            P = P + np.eye(23) * 1e-2
            x, P, info = g.scan(scans[k], x, P)
            out.append((x.copy(), info["n_down"], info["n_eff"]))
        g.sync()
        return out

    def run_in_place():
        """scan_into: the same entry point without the per-call arrays / dict (bench.py's timed loop)."""
        g, o, prior = _pair(small_world)
        x = np.array(prior.to_vec(), np.float64); P = np.array(eskf.init_P(), np.float64)
        info = lsdreg.capi.LioInfo()
        out = []
        for k in range(4):
            P += np.eye(23) * 1e-2
            assert g.scan_into(scans[k], x, P, info) >= 0
            out.append((x.copy(), info.n_down, info.n_eff))
        g.sync()
        return out

    ref = run("serial")
    for (xa, na, ea), (xb, nb, eb) in zip(ref, run_in_place()):
        assert na == nb and ea == eb
        np.testing.assert_array_equal(xa, xb)
    for mode in ("pipelined", "decoy"):
        got = run(mode)
        for (xa, na, ea), (xb, nb, eb) in zip(ref, got):
            assert na == nb and ea == eb
            np.testing.assert_array_equal(xa, xb)


def test_degenerate_scene_projection():
    """laserMapping.cpp:934-980 on the device: a ground-plane-only scene (tests/scenes.py) is flagged degenerate in every
    evaluation — the host eigenvalue certificate fails, lio_degen_kernel computes the per-direction sums, the normal
    equations are projected with mat_p — and the posterior equals the restated pipeline's, which
    tests/test_oracle_degenerate.py pins to laserMapping.cpp compiled unmodified (3e-9 m)."""
    import lsdreg
    import scenes
    from oracle import eskf
    from oracle.lio import OracleLio
    w = scenes.plane_world()
    prior = eskf.State(); prior.rot = eskf.R_to_quat(w["Rprior"]); prior.pos = w["tprior"].copy()
    g = lsdreg.LioFrontend(map_log2_lines=18)
    g.map.insert(w["map"], 0); g.set_next_id(w["map"].shape[0])
    o = OracleLio(18, expected_cells=1 << 18, stale_neighbours=True)
    o.add_map_points(w["map"])
    # single evaluation first: flag, projected normal equations
    n = g.load_scan(w["scan"])
    body = g.get_down()
    o.near_xyz = np.zeros((n, 5, 3), np.float32); o.near_ids = np.full((n, 5), -1, np.int32)
    o.near_cnt = np.zeros(n, np.int32); o.selected = np.ones(n, np.uint8)
    o.world = np.zeros((n, 4), np.float32); o.plane = np.zeros((n, 4), np.float32)
    ro = o._hmodel(body, prior, True)
    rg = g.linearize(prior.to_vec(), True)
    assert rg["degenerate"] == 1 and o.last["degenerate"] == 1 and rg["n_eff"] == ro["n"] > 3000
    np.testing.assert_allclose(rg["HTH"], o.last["HTH6"], rtol=1e-9, atol=1e-7)
    np.testing.assert_allclose(rg["HTh"], o.last["HTh6"], rtol=1e-9, atol=1e-7)
    # whole scan through lsd_lio_scan vs the restated fastlio_main pass, same downsampled cloud
    g2 = lsdreg.LioFrontend(map_log2_lines=18)
    g2.map.insert(w["map"], 0); g2.set_next_id(w["map"].shape[0])
    x, P, info = g2.scan(w["scan"], prior.to_vec(), eskf.init_P())
    o2 = OracleLio(18, expected_cells=1 << 18, stale_neighbours=True)
    o2.add_map_points(w["map"])
    r = o2.process_scan(g2.get_down(), prior, eskf.init_P(), downsample=False)
    xo = o2.x.to_vec()
    assert info["degenerate"] == 1 and info["iterations"] == r["iters"] and info["n_eff"] == r["log"][-1]["n_eff"]
    assert np.abs(x[0:3] - xo[0:3]).max() < POS_TOL and _rot_err(x[3:7], xo[3:7]) < ROT_TOL
    np.testing.assert_allclose(x, xo, atol=1e-7)
    np.testing.assert_allclose(P, o2.P, rtol=1e-4, atol=1e-8)      # unobservable directions: entries of 1e-10 are rounding noise
    assert np.abs(x[:2] - w["tprior"][:2]).max() < 1e-3 and abs(x[2] - w["tgt"][2]) < 5e-3   # x / y unobservable: untouched
    assert abs(info["n_added"] - r["added"]) <= 3


@pytest.mark.parametrize("per_voxel,nearby", [(8, 18), (14, 18), (30, 18), (3, 74), (9, 6)])
def test_reference_order_on_crowded_voxels(per_voxel, nearby):
    """lsd_lio_set_reference_order on maps the bench never builds: 14 and 30 points per voxel (KNNPointByCondition's per-voxel
    nth_element + truncation, overflow lines beyond the 7 points of a cell line, more candidates than the search's list
    holds -> the counted canonical fallback), exact duplicates (distance ties), NEARBY74 / NEARBY6 — Nearest_Points rows
    against the oracle's reference-order k-NN (pinned id for id to the compiled iVox) position by position."""
    import lsdreg
    from oracle import eskf
    from oracle import oracle as O
    rng = np.random.default_rng([11, per_voxel, nearby])
    side = 6.0
    n_map = int(per_voxel * (2 * side / 0.5) ** 2 * 4)             # a slab 2 m thick
    m = np.zeros((n_map, 4), np.float32)
    m[:, 0:2] = rng.uniform(-side, side, (n_map, 2)); m[:, 2] = rng.uniform(-1.0, 1.0, n_map)
    m[n_map // 2:n_map // 2 + 500, :3] = m[:500, :3]               # duplicates
    g = lsdreg.LioFrontend(map_log2_lines=18, ivox_nearby=nearby, max_points=20000)
    g.set_reference_order(True)
    for a in range(0, n_map, n_map // 3 + 1):
        g.map.insert(np.ascontiguousarray(m[a:a + n_map // 3 + 1]), a)
    po = O.OracleIvox(0.5, nearby, 1 << 16)
    for a in range(0, n_map, n_map // 3 + 1):
        po.add(np.ascontiguousarray(m[a:a + n_map // 3 + 1]), a)
    q = np.zeros((3000, 4), np.float32)
    q[:, 0:2] = rng.uniform(-side - 1, side + 1, (3000, 2)); q[:, 2] = rng.uniform(-2.5, 2.5, 3000)
    n = g.load_scan(q, downsample=False)
    assert n == 3000
    x = eskf.State()
    g.linearize(x.to_vec(), True)
    mt = g.get_matches()
    ids, d2, xyz, cnt = po.knn(np.ascontiguousarray(mt["world"][:, :4]), 5, 5.0, reference_order=True)
    fb = g.reference_order_fallbacks()
    assert (mt["cnt"] == cnt).all()
    same = (mt["idx"] == ids).all(1)
    if nearby == 6 or per_voxel == 8:
        assert fb == 0                                              # ~63 / ~150 candidates per query: inside the list's 256
    assert (~same).sum() <= fb                                      # only rows that fell back may differ in order
    assert (np.sort(mt["idx"], 1) == np.sort(ids, 1)).all(1).mean() > 0.995   # and even those hold the same neighbours up to ties at the fifth place
    if per_voxel == 30:
        assert fb > 0


def test_reference_order_truncates_crowded_voxels_in_short_sequences():
    """A sparse map (well under 32 candidates per query: the warp-cooperative replay) with clusters of 7-12 points packed into
    single voxels: KNNPointByCondition's per-voxel nth_element + truncation (ivox3d_node.hpp:118-123) inside the warp path,
    including two crowded voxels in one stencil and exact duplicates inside a cluster."""
    import lsdreg
    from oracle import eskf
    from oracle import oracle as O
    rng = np.random.default_rng(77)
    side = 8.0
    base = np.zeros((3000, 4), np.float32)
    base[:, 0:2] = rng.uniform(-side, side, (3000, 2)); base[:, 2] = rng.uniform(-0.6, 0.6, 3000)
    centres = (np.floor(rng.uniform(-side + 1, side - 1, (120, 3)) * [1, 1, 0.1] / 0.5) * 0.5 + 0.25).astype(np.float32)
    centres[60:] = centres[:60] + np.float32([0.5, 0, 0])                  # pairs of neighbouring crowded voxels
    clusters = []
    for c in centres:
        k = int(rng.integers(7, 13))
        pts = c + rng.uniform(-0.2, 0.2, (k, 3)).astype(np.float32)
        pts[1] = pts[0]                                                     # a duplicate: a tie inside the voxel
        clusters.append(pts)
    cl = np.concatenate(clusters)
    m = np.concatenate([base, np.concatenate([cl, np.zeros((cl.shape[0], 1), np.float32)], 1)])
    m = np.ascontiguousarray(m[rng.permutation(m.shape[0])])
    g = lsdreg.LioFrontend(map_log2_lines=16, ivox_nearby=18, max_points=20000)
    g.set_reference_order(True)
    po = O.OracleIvox(0.5, 18, 1 << 14)
    for a in range(0, m.shape[0], 1500):
        g.map.insert(np.ascontiguousarray(m[a:a + 1500]), a); po.add(np.ascontiguousarray(m[a:a + 1500]), a)
    q = np.zeros((4000, 4), np.float32)
    q[:2000, :3] = centres[rng.integers(0, 120, 2000)] + rng.uniform(-0.7, 0.7, (2000, 3)).astype(np.float32)
    q[2000:, 0:2] = rng.uniform(-side, side, (2000, 2)); q[2000:, 2] = rng.uniform(-1, 1, 2000)
    assert g.load_scan(q, downsample=False) == 4000
    g.linearize(eskf.State().to_vec(), True)
    mt = g.get_matches()
    qq = np.ascontiguousarray(mt["world"][:, :4])
    ids, d2, xyz, cnt = po.knn(qq, 5, 5.0, reference_order=True)
    allc = po.knn(qq, 64, 5.0)[3]
    assert (allc <= 32).mean() > 0.6 and (allc > 5).mean() > 0.5            # most queries take the warp path, the rest the serial replay
    assert g.reference_order_fallbacks() == 0
    assert (mt["cnt"] == cnt).all()
    assert (mt["idx"] == ids).all()


def test_device_nth_element_is_the_oracles():
    """lsd_debug_nth_element — std::nth_element as the search kernel replays it (warp-cooperative for up to 32 elements, serial
    else and past introselect's depth limit) — against the oracle's restatement, itself pinned to std::nth_element
    (tests/test_oracle_golden.py): the same permutation on every sequence, every path taken."""
    import ctypes as C
    import lsdreg
    from oracle import oracle as O
    import test_oracle_golden as T
    paths = {1: 0, 2: 0, 3: 0}

    def check(d, first, nth, last):
        n = d.shape[0]
        want = np.arange(n, dtype=np.int32)
        O.port.orc_nth_element(C.c_void_p(d.ctypes.data), C.c_void_p(want.ctypes.data), n, first, nth, last)
        got, path = lsdreg.capi.debug_nth_element(d, first, nth, last)
        assert (got == want).all(), (n, first, nth, last, path)
        paths[path] += 1
    for d, first, nth, last in T._nth_sequences(np.random.default_rng(8), 1500):
        check(d, first, nth, last)
    for d, first, nth, last in T._depth_limit_sequences():
        check(d, first, nth, last)
    assert paths[1] > 300 and paths[3] > 300 and paths[2] >= 8, paths
