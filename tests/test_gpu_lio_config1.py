"""GPU parity at BASELINE.json config[1] scale: the bench workload itself (bench.make_step: ~100 k-return 64-beam scan vs the
10.1 M-point map, full iterate-to-converge, every step in another block) through lsd_lio_scan, against

  (a) laserMapping.cpp COMPILED UNMODIFIED (oracle/_ref/libref_fastlio.so, RefFastLioBench.process_scan — the very code
      bench.py --impl reference times; its posteriors and counts are stored in tests/golden/config1_ref.npz by
      tests/golden/make_golden_config1.py): posterior pose within the north_star's 1e-4 m / 1e-5 rad on every step, same
      feats_down_size, same effective-point count to a handful of gate flips (the compiled reference keeps
      std::nth_element's neighbour order, esti_plane's QR is order-sensitive in fp32 — DESIGN.md section 4);
  (b) the plain-C port of iVox on the SAME 10 M-point map: bit-exact neighbour ids for every query of the scan's first
      search, on the shared downsampled cloud.

Both sides start from the same map and register the same scans in the same order, map_incremental included, so step s sees
the map the steps before it left behind.  The GPU run uses the full 13 x 13-block map the golden vectors were made on."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_STEPS = 6
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "config1_ref.npz")


@pytest.mark.parametrize("ref_order", [False, True])
def test_bench_steps_pose_parity_with_the_compiled_reference(ref_order):
    """ref_order (lsd_lio_set_reference_order, the default): neighbours in the order IVox::GetClosestPoint returns them, esti_plane
    in Eigen's summation order, the voxel grid's centroids as the restated pcl::VoxelGrid's sequential fp32 sums: nothing separates
    the product from laserMapping.cpp any more but the order of the double-precision normal-equation sums and the Schur form of
    the Kalman gain.  Bars then: effective-point counts and map sizes EQUAL, neighbour ids equal position by position, posterior
    within 1e-9 m / 1e-10 rad (measured under the emulator: 7e-15 m / 1e-16 rad).  ref_order False: rows sorted by distance,
    the north_star's 1e-4 m / 1e-5 rad."""
    import bench
    import lsdreg
    from lsdreg import synth
    from oracle import eskf
    from oracle import oracle as O
    gold = np.load(GOLDEN)
    assert int(gold["x"].shape[0]) >= N_STEPS
    nb = bench.BLOCKS_X
    m = synth.block_map(bench.MAP_SEED, nb, nb, bench.SPACING)
    assert m.shape[0] > 10_000_000 and m.shape[0] == int(gold["map_points"])
    g = lsdreg.LioFrontend(map_log2_lines=25, max_scan_points=131072, max_points=100000, async_map_insert=1)
    g.map.insert(m, 0); g.set_next_id(m.shape[0])
    g.set_reference_order(ref_order)
    port = O.OracleIvox(0.5, 18, 1 << 24)
    port.add(np.ascontiguousarray(m[:, :3]), 0)
    P0 = eskf.init_P()
    worst = np.zeros(2)
    for s in range(N_STEPS):
        scan, Rgt, tgt, Rp, tp = bench.make_step(s)
        prior = eskf.State(); prior.rot = eskf.R_to_quat(Rp); prior.pos = tp.copy()
        if s == 0:
            # (b) the first search of the scan on the device vs the port's iVox, same queries, same 10 M-point map
            n = g.load_scan(scan)
            g.linearize(prior.to_vec(), True)
            mt = g.get_matches()
            oi, od, _, oc = port.knn(np.ascontiguousarray(mt["world"][:, :4]), 5, 5.0, reference_order=ref_order)
            assert (mt["cnt"] == oc).all() and (oc == 5).mean() > 0.5
            found = oc > 0                      # rows that found nothing keep what they held (empty on a first scan)
            assert (mt["idx"][found] == oi[found]).all()
            assert (mt["idx"][~found] == -1).all()
        x, P, info = g.scan(scan, prior.to_vec(), P0)
        xr, Pr = eskf.State.from_vec(gold["x"][s]), gold["P"][s]
        n_down_ref, *cnt = (int(v) for v in gold["counts"][s])
        c = dict(zip(("n_down", "n_eff", "degenerate", "map_cells"), cnt))
        assert info["status"] == lsdreg.OK and info["n_down"] == n_down_ref == c["n_down"], (s, info, c)
        assert abs(info["n_eff"] - c["n_eff"]) <= (0 if ref_order else max(3, c["n_eff"] // 500)), (s, info["n_eff"], c["n_eff"])
        assert info["degenerate"] == c["degenerate"] == 0
        d = np.abs(eskf.State.from_vec(x).boxminus(xr))
        worst = np.maximum(worst, [d[0:3].max(), d[3:6].max()])
        assert d[0:3].max() < (1e-9 if ref_order else 1e-4) and d[3:6].max() < (1e-10 if ref_order else 1e-5), (s, d[:6])
        assert np.abs(x[:3] - tgt).max() < 0.05          # and both sit on the ground truth (2 cm range noise)
        sd = np.sqrt(np.abs(np.diag(Pr)))
        assert (np.abs(P - Pr) <= 1e-3 * np.outer(sd, sd) + 1e-14).all(), s
    g.sync()
    st = g.map.stats()
    assert abs(int(st["cells"]) - c["map_cells"]) <= (0 if ref_order else 8 * N_STEPS), (st, c)     # both maps grew by the same inserts (a gate flip moves a point or two)
    if ref_order:
        assert g.reference_order_fallbacks() == 0
    print(f"config[1] parity vs laserMapping.cpp (reference order {ref_order}): worst |dpos| = {worst[0]:.2e} m, |drot| = {worst[1]:.2e} rad over {N_STEPS} steps")
