"""GPU parity: iVox's capacity / LRU eviction (IVox::AddPoints, ivox3d.h:231-256) — lsd_map_enable_lru — against the
COMPILED reference iVox (oracle/_ref/libref_lio.so) on a stream that crosses the capacity many times over: a sensor
driving away (travel distance grows, old voxels age past max_distance and fall off the back of the LRU list), then
coming back over ground it has forgotten.  Bars: the same number of voxels alive after every batch; the same neighbours
(as sets: the reference returns nearest-first-then-nth_element order) for queries all over the visited ground, old
(evicted) ground included."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_lru_eviction_matches_compiled_ivox():
    import lsdreg
    from oracle import oracle as O
    if not O.HAVE_REF:
        pytest.skip("oracle/_ref/libref_lio.so not built (needs /root/reference at build time)")
    rng = np.random.default_rng(3)
    CAP = 4000
    g = lsdreg.HashVoxelMap(0.5, 16)
    g.enable_lru(CAP, 100.0)
    r = O.RefIvox(0.5, 18, CAP)
    xs = np.concatenate([np.arange(0, 260, 2.0), np.arange(260, -2, -4.0)])       # out 260 m, back to the start
    next_id, dist, prev = 0, 0.0, xs[0]
    inserted = []
    for k, x in enumerate(xs):
        dist += abs(x - prev); prev = x
        n = int(rng.integers(300, 900))
        pts = np.zeros((n, 4), np.float32)
        pts[:, 0] = x + rng.uniform(-12, 12, n); pts[:, 1] = rng.uniform(-8, 8, n); pts[:, 2] = rng.uniform(0, 1.5, n)
        if k % 7 == 3:                                   # now and then the same voxels twice (touches without new voxels); no exact duplicates:
            pts[n // 2:, :3] = pts[:n - n // 2, :3] + rng.uniform(-2e-3, 2e-3, (n - n // 2, 3)).astype(np.float32)   # ties at the 5th place are nth_element's call
        g.set_travel_distance(dist)
        g.insert(pts, next_id)
        r.add(pts, next_id, dist)
        inserted.append(pts[:, :3].astype(np.float64))       # row = id
        next_id += n
        st = g.stats()
        assert st["cells"] == r.num_cells, (k, st, r.num_cells)
        if O.HAVE_REF_IVOX_DUMP:
            assert st["points"] == r.num_points, (k, st, r.num_points)
        if k % 9 == 0 or k == len(xs) - 1:
            q = np.zeros((600, 4), np.float32)
            q[:, 0] = rng.uniform(xs.min() - 12, xs.max() + 12, 600); q[:, 1] = rng.uniform(-8, 8, 600); q[:, 2] = rng.uniform(0, 1.5, 600)
            q[:200, 0] = x + rng.uniform(-12, 12, 200)
            gi, gd, gc = g.knn(q, k=5, max_sq=5.0, stencil=18)
            ri, rx, rc = r.knn(q, 5, 5.0)
            assert (gc == rc).all(), k
            # the sets may differ only through a distance tie at the k-th place (a tie in float32: both sides rank by float
            # d2).  Both rows' d2 are evaluated here, in double, from the neighbours' coordinates: the rows agree on every
            # neighbour clearly nearer than the k-th distance, and the neighbours that differ sit at that distance to
            # within float32 rounding
            allp = np.concatenate(inserted)
            assert (allp[np.where(ri >= 0, ri, 0)][ri >= 0] == rx[ri >= 0]).all()
            for qi, (a, b, c) in enumerate(zip(gi, ri, gc)):
                if set(a[:c]) == set(b[:c]):
                    continue
                da = ((allp[a[:c]] - q[qi, :3]) ** 2).sum(-1)
                db = ((allp[b[:c]] - q[qi, :3]) ** 2).sum(-1)
                kth, tol = da.max(), 1e-6 * da.max()
                assert abs(db.max() - kth) <= tol, (k, qi, da, db)
                assert set(a[:c][da < kth - tol]) == set(b[:c][db < kth - tol]), (k, qi, a[:c], b[:c])
                for d in np.r_[da[~np.isin(a[:c], b[:c])], db[~np.isin(b[:c], a[:c])]]:
                    assert abs(d - kth) <= tol, (k, qi, da, db)
    n_ev = g.evict()
    assert n_ev > 3 * CAP, (n_ev, st)       # the capacity was crossed many times over (voxels younger than max_distance are never dropped: cells may exceed it)
    assert g.stats()["dropped"] == 0
    # the retired lines did not pile up: the table of 65 536 lines was rebuilt along the way and still answers
    assert g.saturated() == (False, 0)


def test_lio_with_lru_keeps_the_map_at_capacity(small_world):
    """The LIO front-end with the reference's eviction on (tiny capacity): scans are registered as before, the map stops at
    the capacity, and the evictions happen with the travel distance the front-end keeps itself (laserMapping.cpp:1289-1291)."""
    import lsdreg
    from lsdreg import synth
    from oracle import eskf
    g = lsdreg.LioFrontend(map_log2_lines=18)
    g.map.enable_lru(9000, 0.3)                         # 0.3 m: every voxel older than one step is old enough
    x = lsdreg.make_state(pos=small_world["tgt"], rot_xyzw=eskf.R_to_quat(small_world["Rgt"]))
    P = lsdreg.init_cov()
    cells = []
    for k in range(6):
        Rk = small_world["Rgt"] @ synth.rot_from_rpy(0, 0, 0.02 * k)
        tk = small_world["tgt"] + np.array([0.4 * k, 0.1 * k, 0.0])
        scan = synth.scan64(10 + k, 250, Rk, tk)
        P = P + np.eye(23) * 1e-2
        x, P, info = g.scan(scan, x, P)
        assert info["status"] in (lsdreg.OK, lsdreg.MAP_SEEDED)
        cells.append(g.map.stats()["cells"])
        if k:
            assert np.abs(x[:3] - tk).max() < 0.1
    assert max(cells) <= 9001 and cells[-1] >= 8999 and g.map.evict() > 1000, (cells, g.map.evict())
