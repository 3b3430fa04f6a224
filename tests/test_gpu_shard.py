"""GPU: tile-sharded LIO (SURVEY.md §8e).  Two ranks are emulated on ONE device — two handles in one
process, driven by two threads (ctypes releases the GIL) — so the peer-memory all-reduce fused into
the reduction kernel and the halo exchange run for real on the single-GPU test box.  Bars: every
rank's shard holds exactly the points relevant to it; the sharded pose equals the unsharded pose to
1e-9 (sums are folded in rank order, not in the single-GPU block order)."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run_threads(fns):
    out, err = [None] * len(fns), []

    def w(i):
        try:
            out[i] = fns[i]()
        except Exception as e:  # pragma: no cover
            err.append(e)

    th = [threading.Thread(target=w, args=(i,)) for i in range(len(fns))]
    [t.start() for t in th]
    [t.join(timeout=120) for t in th]
    assert not any(t.is_alive() for t in th), "sharded ranks deadlocked"
    if err:
        raise err[0]
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_ranks_match_single_gpu(small_world, world):
    import lsdreg
    from lsdreg import shard
    from oracle import eskf
    m, scan = small_world["map"], small_world["scan"]
    prior = lsdreg.make_state(pos=small_world["tprior"], rot_xyzw=eskf.R_to_quat(small_world["Rprior"]))
    P0 = lsdreg.init_cov()
    single = lsdreg.LioFrontend(map_log2_lines=20)
    single.map.insert(m, 0); single.set_next_id(m.shape[0])
    single.load_scan(scan)
    xs, Ps, infos = single.update(prior, P0)

    lios = [lsdreg.LioFrontend(map_log2_lines=20) for _ in range(world)]
    blobs = np.stack([l.shard_export(r, world, shard.TILE_CELLS, 1) for r, l in enumerate(lios)])
    for l in lios:
        l.shard_connect(blobs)
    cells = shard.cell_of(m[:, :3])
    for r, l in enumerate(lios):
        l.map.insert(m, 0); l.set_next_id(m.shape[0])
        st = l.map.stats()
        assert st["points"] == int(shard.relevant(cells, r, world).sum())   # host mirror == device ownership
        assert st["points"] < m.shape[0]
    res = _run_threads([lambda l=l: l.scan(scan, prior, P0) for l in lios])
    for x, P, info in res:
        np.testing.assert_allclose(x, xs, rtol=0, atol=1e-9)
        np.testing.assert_allclose(P, Ps, rtol=1e-4, atol=1e-12)
        assert info["n_eff"] == infos["n_eff"] and info["iterations"] == infos["iterations"]
    for r in range(1, world):
        np.testing.assert_array_equal(res[0][0], res[r][0])                   # ranks agree bit for bit
    # map_incremental (+ halo exchange): each point's owner decides; rank r inserts exactly the added points whose home
    # voxel is relevant to it (its own and its halo's) and again holds exactly its relevant points.  The decision per
    # point against the single handle at the same state is tests/test_gpu_shard_contents.py.
    w = lios[0].get_matches()["world"][:, :3]
    assert all(np.array_equal(l.get_matches()["world"][:, :3], w) for l in lios[1:])
    wcells = shard.cell_of(w)
    owner = shard.tile_owner(wcells[:, 0], wcells[:, 1], shard.TILE_CELLS, world)
    added = np.choose(owner, [l.get_map_flags()[0] for l in lios]) > 0
    assert added.any()
    for r, l in enumerate(lios):
        assert res[r][2]["n_added"] == int((added & shard.relevant(wcells, r, world)).sum())
        assert l.map.stats()["points"] == int(shard.relevant(cells, r, world).sum()) + res[r][2]["n_added"]


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_ndt_matches_single_gpu(world):
    """Row C3 of SURVEY.md section 8e: the NDT target voxelised per x-y tile on its owner, [H, b, err] all-reduced inside the
    cost kernel.  Ranks are emulated on one device (two / three handles, one thread each).  Bars: the voxel counts of the
    shards partition the unsharded map; one cost evaluation equals the unsharded one to 1e-12 relative (same fp32
    per-point terms, double sums in another order); align() returns the same pose to 1e-9 with the same iteration count
    and flag; all ranks agree bit for bit."""
    import lsdreg
    from lsdreg import synth
    m = synth.block_map(1, 1, 1, 0.25)
    m[:, :2] -= np.array([60, 40], np.float32)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = np.array([1.0, -2.0, 1.8])
    scan = synth.scan64(2, 200, Rgt, tgt + np.array([60, 40, 0]))[::2].copy()
    dR, dt = synth.perturb(5, 0.5, 3.0)
    guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
    single = lsdreg.Matcher("NDT_CUDA")
    single.set_target(m); single.set_source(scan)
    e1, H1, b1, nc1 = single.cost(guess)
    T1 = single.align(guess); T1d, _ = single.final()
    it1, cv1 = single.iterations, single.converged

    ranks = [lsdreg.Matcher("NDT_CUDA") for _ in range(world)]
    blobs = np.stack([r.shard_export(k, world, 8) for k, r in enumerate(ranks)])      # 8-voxel tiles: many tiles in a 120 x 80 m block
    for r in ranks:
        r.shard_connect(blobs)
    for r in ranks:
        r.set_target(m); r.set_source(scan)          # each rank filters the cloud by tile ownership on the device
    nv = [r.stats()["n_voxels"] for r in ranks]
    assert sum(nv) == single.stats()["n_voxels"] and min(nv) > 0, (nv, single.stats())
    res = _run_threads([lambda r=r: r.cost(guess) for r in ranks])
    for e, H, b, nc in res:
        assert nc == nc1
        np.testing.assert_allclose(e, e1, rtol=1e-12)
        np.testing.assert_allclose(H, H1, rtol=1e-11, atol=1e-11 * np.abs(H1).max())
        np.testing.assert_allclose(b, b1, rtol=1e-11, atol=1e-11 * np.abs(b1).max())
    assert all(np.array_equal(res[0][1], x[1]) for x in res[1:])                      # rank-ordered fold: bit-identical
    outs = _run_threads([lambda r=r: (r.align(guess), r.final()[0], r.iterations, r.converged) for r in ranks])
    for T, Td, it, cv in outs:
        assert it == it1 and cv == cv1
        np.testing.assert_allclose(Td, T1d, rtol=0, atol=1e-9)
    assert all(np.array_equal(outs[0][1], x[1]) for x in outs[1:])
    with pytest.raises(lsdreg.LsdError):
        ranks[0].fitness(25.0)
    g = lsdreg.Matcher("FAST_GICP")
    with pytest.raises(lsdreg.LsdError):
        g.shard_export(0, 2, 8)
