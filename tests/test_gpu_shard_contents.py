"""GPU: the tile-sharded LIO map, its halo exchange and the sharded NDT target, point by point against the single-GPU
handle.  Ranks are emulated on one device as in tests/test_gpu_shard.py: one handle per rank, each collective call issued
on every rank of the world from its own thread.  The sharded ranks and the single handle are driven at the SAME states
(linearize / map_incremental, not update), so every comparison is exact:
  * map contents: rank r's dump is the single map's dump restricted to the voxels shard.relevant(., r) holds — the same
    voxel keys and, per voxel, the same multiset of (x, y, z, id) bits — after the initial insert and after every
    map_incremental (halo copies carry their owner's ids, id_t2 included);
  * search rows: every scan point is resolved by exactly one rank, the owner of its home voxel, and that rank's row is the
    single handle's bit for bit (count, ids, coordinates, selected flag, plane, world point); the others report cnt = -1;
  * sums: n_eff / degenerate equal, HTH / HTh / res_sum bit-identical across ranks, and the sharded and single sums both
    within m 2^-52 sum|terms| of an exact (math.fsum) sum of the rows;
  * map_incremental: the owner's decision per point is the single handle's;
  * the NDT target: rank r holds exactly the unsharded voxels whose x-y tile it owns, with the same counts and moments.
Small tiles (3, 5 and 13 voxels for halos of 1, 2 and 6) put most voxels in some halo, and the drive crosses x = 0 and
y = 0 so that negative cells and floor division occur.  The stale-rows switch is off on the single handle: a sharded
handle has it off by construction (include/lsdreg.h)."""
import functools
import math

import numpy as np
import pytest

from test_gpu_shard import _run_threads

pytestmark = pytest.mark.gpu

SHIFT = np.array([60.0, 40.0, 0.0])          # block (0, 0) centred on the origin of the map frame
N_SCANS = 15


@functools.lru_cache(maxsize=None)
def _map():
    from lsdreg import synth
    m = synth.block_map(1, 1, 1, 0.5)
    m[:, :2] -= SHIFT[:2].astype(np.float32)
    return m


@functools.lru_cache(maxsize=None)
def _drive(n):
    """n scans along a path that crosses x = 0 and y = 0 several times (map frame) -> [(R, t, body scan)]."""
    from lsdreg import synth
    out = []
    for k in range(n + 1):
        s = k / n
        t = np.array([-7.0 + 14.0 * s, 3.0 * math.sin(7.0 * s), 1.8])
        R = synth.rot_from_rpy(0.01 * math.sin(3 * s), -0.015, 0.3 + 1.2 * s)
        out.append((R, t, synth.scan64(40 + k, 100, R, t + SHIFT)))
    return out


def _state(R, t, k=0):
    """A common state near the true pose: a small perturbation fixed per k."""
    import lsdreg
    from lsdreg import synth
    from oracle import eskf
    dR, dt = synth.perturb(100 + k, 0.08, 0.4)
    return lsdreg.make_state(pos=t + dt, rot_xyzw=eskf.R_to_quat(R @ dR))


# ------------------------------------------------------------------ read-backs
def _contents(g):
    """Live points as rows (voxel x, y, z, x bits, y bits, z bits, id) sorted lexicographically: equal arrays <=> the same
    voxel keys and per voxel the same multiset of points.  Asserts stats() against the dump."""
    d = g.dump()
    st = g.stats()
    assert not d["tombstone"].any()
    rows = np.concatenate([d["voxel"].astype(np.int64), np.ascontiguousarray(d["xyz"]).view(np.uint32).astype(np.int64),
                           d["id"].astype(np.int64)[:, None]], 1)
    rows = rows[np.lexsort(rows.T[::-1])]
    assert st["points"] == len(rows) and st["cells"] == len(np.unique(rows[:, :3], axis=0)), st
    return rows


def _assert_shards(single, ranks, world, tile, reach, what):
    from lsdreg import shard
    full = _contents(single.map)
    seen = np.zeros(len(full), int)
    for r, l in enumerate(ranks):
        rel = shard.relevant(full[:, :3].astype(np.int32), r, world, tile, reach)
        want, got = full[rel], _contents(l.map)
        if not np.array_equal(got, want):
            a = {tuple(x) for x in got.tolist()}
            b = {tuple(x) for x in want.tolist()}
            raise AssertionError(f"{what}: rank {r} of {world}: {len(a - b)} points only on the shard {sorted(a - b)[:3]}, "
                                 f"{len(b - a)} missing {sorted(b - a)[:3]}")
        seen += shard.owns(full[:, :3].astype(np.int32), r, world, tile)
    assert (seen == 1).all()
    return full


def _owners(world_xyz, world, tile):
    from lsdreg import shard
    c = shard.cell_of(world_xyz[:, :3])
    return shard.tile_owner(c[:, 0], c[:, 1], tile, world), c


def _same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _assert_rows(single, ranks, world, tile, what, owner=None):
    """Owned rows equal the single handle's bit for bit; every point resolved by exactly its owner — the owner of its home
    voxel at the state of the search (pass it for the evaluations that reuse the search's rows).  -> (matches, owner)"""
    ms = single.get_matches()
    mr = [l.get_matches() for l in ranks]
    for r, m in enumerate(mr):
        assert (m["world"][:, :3].view(np.uint32) == ms["world"][:, :3].view(np.uint32)).all(), (what, r)
    if owner is None:
        owner, _ = _owners(ms["world"], world, tile)
    resolved = np.stack([m["cnt"] != -1 for m in mr])
    assert (resolved.sum(0) == 1).all() and (resolved.argmax(0) == owner).all(), what
    assert (ms["cnt"] >= 0).all()
    for r, m in enumerate(mr):
        o = owner == r
        bad = np.nonzero(o & (m["cnt"] != ms["cnt"]))[0]
        assert not len(bad), f"{what}: rank {r}: cnt differs at {bad[:8]}: {m['cnt'][bad[:8]]} vs {ms['cnt'][bad[:8]]}"
        live = o[:, None] & (np.arange(5)[None, :] < ms["cnt"][:, None])
        assert (m["idx"][live] == ms["idx"][live]).all(), (what, r)
        assert (m["xyz"][live].view(np.uint32) == ms["xyz"][live].view(np.uint32)).all(), (what, r)
        bad = np.nonzero(o & (m["selected"] != ms["selected"]))[0]
        assert not len(bad), f"{what}: rank {r}: selected differs at {bad[:8]}"
        assert not m["selected"][~o].any(), (what, r)
        sel = o & (ms["selected"] > 0)
        assert _same_bits(m["plane"][sel], ms["plane"][sel]).all(), (what, r)
    return ms, owner


def _rows_of(g, ms, x):
    """Jacobian rows and residuals of the selected points (laserMapping.cpp:903-932), rebuilt in double from the read-back."""
    from oracle import eskf
    body = g.get_down()[:, :3].astype(np.float64)
    sel = ms["selected"] > 0
    R = eskf.quat_to_R(x[3:7])
    nrm = ms["plane"][sel, :3].astype(np.float64)
    c = nrm @ R                                               # R^T n, one row per point
    lp = body[sel]
    hx = np.concatenate([nrm, np.cross(lp, c)], 1)
    return hx, -ms["plane"][sel, 3].astype(np.float64)


def _assert_sum_bar(got, hx, h, what):
    m = len(h)
    for a in range(6):
        for c in range(6):
            t = hx[:, a] * hx[:, c]
            assert abs(got["HTH"][a, c] - math.fsum(t)) <= m * 2.0 ** -52 * math.fsum(np.abs(t)), (what, a, c)
        t = hx[:, a] * h
        assert abs(got["HTh"][a] - math.fsum(t)) <= m * 2.0 ** -52 * math.fsum(np.abs(t)), (what, a)
    assert abs(got["res_sum"] - math.fsum(np.abs(h))) <= m * 2.0 ** -52 * math.fsum(np.abs(h)), what


def _linearize_all(single, ranks, x, search, what):
    rs = single.linearize(x, search)
    rr = _run_threads([lambda l=l: l.linearize(x, search) for l in ranks])
    for r in rr:
        assert r["n_eff"] == rs["n_eff"] and r["degenerate"] == rs["degenerate"] and r["status"] == rs["status"], what
        for k in ("HTH", "HTh"):
            assert np.array_equal(r[k], rr[0][k]), (what, k)
        assert r["res_sum"] == rr[0]["res_sum"], what
    if rs["n_eff"] > 0 and not rs["degenerate"]:
        ms = single.get_matches()
        hx, h = _rows_of(single, ms, x)
        assert len(h) == rs["n_eff"]
        _assert_sum_bar(rs, hx, h, what + " single")
        _assert_sum_bar(rr[0], hx, h, what + " sharded")
    return rs, rr


# ------------------------------------------------------------------ 1. the LIO shard, scan by scan
CASES = {   # stencil (None = knn_mode_exact), reach, tile, reference order, seeding scan on an empty map, ekf_inited
    "nearby18_ref": (18, 1, 3, True, False, True),
    "nearby18_canonical": (18, 1, 3, False, False, True),
    "nearby74": (74, 2, 5, True, False, True),
    "exact": (None, None, 13, False, False, True),
    "seeded": (18, 1, 3, True, True, True),
    "ekf_not_inited": (18, 1, 3, True, False, False),
}


def _frontends(case, world):
    import lsdreg
    from lsdreg import shard
    stencil, reach, tile, ref, seeded, inited = CASES[case]
    kw = dict(map_log2_lines=18) if stencil is not None else dict(map_log2_lines=18, knn_mode_exact=1)
    if stencil is not None:
        kw["ivox_nearby"] = stencil
    if reach is None:
        reach = shard.exact_reach(0.5)
    single = lsdreg.LioFrontend(**kw)
    single.set_stale_rows(False)
    ranks = [lsdreg.LioFrontend(**kw) for _ in range(world)]
    blobs = np.stack([l.shard_export(r, world, tile, reach) for r, l in enumerate(ranks)])
    for l in ranks:
        l.shard_connect(blobs)
    for l in [single] + ranks:
        l.set_reference_order(ref)
        l.set_ekf_inited(inited)
    return single, ranks, tile, reach, ref, seeded, inited


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", list(CASES))
def test_sharded_lio_scan_by_scan(case, world):
    import lsdreg
    from lsdreg import shard
    single, ranks, tile, reach, ref, seeded, inited = _frontends(case, world)
    allh = [single] + ranks
    m = _map()
    drive = _drive(N_SCANS)
    P0 = lsdreg.init_cov()
    k0 = 0
    if seeded:
        R, t, body = drive[0]
        x = _state(R, t)
        for l in allh:
            l.set_next_id(7)
        xs, _, info = single.scan(body, x, P0)
        out = _run_threads([lambda l=l: l.scan(body, x, P0) for l in ranks])
        assert info["status"] == lsdreg.MAP_SEEDED and all(o[2]["status"] == lsdreg.MAP_SEEDED for o in out)
        assert (single.get_map_flags()[0] == 1).all()
        _assert_shards(single, ranks, world, tile, reach, "seeded map")
        k0 = 1
    else:
        for l in allh:
            l.map.insert(m, 0)
            l.set_next_id(m.shape[0])
        full = _assert_shards(single, ranks, world, tile, reach, "initial map")
        assert (full[:, 0] < 0).any() and (full[:, 1] < 0).any()
    halo_flags = np.zeros(3, int)         # decisions 0 / 1 / 2 on points whose home voxel sits in another rank's halo
    n_owned = np.zeros(world, int)
    for k in range(k0, N_SCANS):
        R, t, body = drive[k]
        n = single.load_scan(body)
        assert all(l.load_scan(body) == n for l in ranks)
        x = _state(R, t, k)
        _linearize_all(single, ranks, x, True, f"scan {k} search")
        ms, owner = _assert_rows(single, ranks, world, tile, f"scan {k} search")
        n_owned += np.bincount(owner, minlength=world)
        for j in (1, 2):                  # reuse evaluations at other states: the rows of the search, planes refitted nowhere
            xj = _state(R, t, 1000 * j + k)
            _linearize_all(single, ranks, xj, False, f"scan {k} reuse {j}")
            _assert_rows(single, ranks, world, tile, f"scan {k} reuse {j}", owner)
        # map_incremental at the state of the search: a rank decides the points whose rows it holds
        na_s = single.map_incremental(x)
        na_r = _run_threads([lambda l=l: l.map_incremental(x) for l in ranks])
        fs = single.get_map_flags()[0]
        fr = [l.get_map_flags()[0] for l in ranks]
        owner2, cells = _owners(single.get_matches()["world"], world, tile)
        assert np.array_equal(owner2, owner)
        union = np.choose(owner, fr)
        bad = np.nonzero(union != fs)[0]
        assert not len(bad), f"scan {k}: map_incremental flags differ at {bad[:8]}: {union[bad[:8]]} vs {fs[bad[:8]]}"
        assert na_s == int((fs > 0).sum())
        for r in range(world):
            rel = shard.relevant(cells, r, world, tile, reach)
            assert na_r[r] == int(((fs > 0) & rel).sum()), (k, r)          # owners' inserts + halo copies
            halo = rel & (owner != r)
            halo_flags += np.bincount(fs[halo], minlength=3)
        if not inited:
            assert (fs == 1).all()
        _assert_shards(single, ranks, world, tile, reach, f"scan {k} after map_incremental")
    print(f"{case} world {world}: owned points per rank {n_owned.tolist()}, halo decisions 0/1/2 {halo_flags.tolist()}")
    assert (n_owned > 0).all()
    assert halo_flags[1] > 0
    if inited:
        assert halo_flags[0] > 0 and halo_flags[2] > 0        # PointNoNeedDownsample copies: the id_t2 ids in halos
    # the whole update() on the last scan: the bars of tests/test_gpu_shard.py
    R, t, body = drive[N_SCANS]
    x = _state(R, t, 5000)
    for l in allh:
        l.load_scan(body)
    xs, _, infos = single.update(x, P0)
    out = _run_threads([lambda l=l: l.update(x, P0) for l in ranks])
    for xr, Pr, info in out:
        np.testing.assert_allclose(xr, xs, rtol=0, atol=1e-9)
        assert info["n_eff"] == infos["n_eff"] and info["iterations"] == infos["iterations"]
        assert np.array_equal(xr, out[0][0])


# ------------------------------------------------------------------ 4. a halo narrower than the search is refused
def test_narrow_halo_is_refused():
    """A reach-1 halo serves NEARBY6/18/26 only.  Everything here is refused on every rank before any collective kernel
    could be launched: exports, stencil switches, batch k-NN queries."""
    import lsdreg
    from lsdreg import shard
    ex = lsdreg.LioFrontend(map_log2_lines=14, knn_mode_exact=1)
    with pytest.raises(lsdreg.LsdError):
        ex.shard_export(0, 2, 13, shard.exact_reach(0.5) - 1)
    wide = lsdreg.LioFrontend(map_log2_lines=14, ivox_nearby=74)
    with pytest.raises(lsdreg.LsdError):
        wide.shard_export(0, 2, 5, 1)
    wide.shard_export(0, 2, 5, 2)
    ranks = [lsdreg.LioFrontend(map_log2_lines=16) for _ in range(2)]
    blobs = np.stack([l.shard_export(r, 2, 3, 1) for r, l in enumerate(ranks)])
    for l in ranks:
        l.shard_connect(blobs)
        l.map.insert(_map(), 0)
        for s in (lsdreg.STENCIL_NEARBY74, lsdreg.STENCIL_EXACT):
            with pytest.raises(lsdreg.LsdError):
                l.set_nearby(s)
        for s in (lsdreg.STENCIL_NEARBY6, lsdreg.STENCIL_NEARBY26, lsdreg.STENCIL_NEARBY18):
            l.set_nearby(s)
    q = np.zeros((64, 4), np.float32)
    q[:, 0] = np.linspace(-3.0, 3.0, 64)
    for s, sq in ((lsdreg.STENCIL_NEARBY74, 5.0), (lsdreg.STENCIL_EXACT, 5.0), (lsdreg.STENCIL_EXACT, 0.0625)):
        with pytest.raises(lsdreg.LsdError):
            ranks[0].map.knn(q, max_sq=sq, stencil=s)
    ranks[0].map.knn(q, stencil=lsdreg.STENCIL_NEARBY18)
    # a reach-2 map serves NEARBY74, and the exact search up to a 0.5 m radius (last shell ceil(0.5 * 2) + 1 = 2)
    m2 = lsdreg.HashVoxelMap(0.5, 14)
    lsdreg.capi.check(lsdreg.capi.lib.lsd_map_set_shard(m2.h, 0, 2, 5, 2))
    m2.insert(_map(), 0)
    m2.knn(q, stencil=lsdreg.STENCIL_NEARBY74)
    m2.knn(q, max_sq=0.0625, stencil=lsdreg.STENCIL_EXACT)
    with pytest.raises(lsdreg.LsdError):
        m2.knn(q, max_sq=0.5, stencil=lsdreg.STENCIL_EXACT)


def test_set_nearby_exact_is_the_exact_search():
    """lsd_lio_set_nearby(EXACT) on a handle in reference-order mode (the default) searches like knn_mode_exact = 1: the
    reference order applies to iVox stencils only, and the exact search has no stencil table to replay it on."""
    import lsdreg
    R, t, body = _drive(N_SCANS)[4]
    x = _state(R, t, 4)
    a = lsdreg.LioFrontend(map_log2_lines=16, knn_mode_exact=1)
    b = lsdreg.LioFrontend(map_log2_lines=16)
    b.set_reference_order(True)
    b.set_nearby(lsdreg.STENCIL_EXACT)
    out = []
    for g in (a, b):
        g.map.insert(_map(), 0)
        g.load_scan(body)
        out.append((g.linearize(x, True), g.get_matches()))
    (ra, ma), (rb, mb) = out
    assert (ma["cnt"] == 5).mean() > 0.5
    for k in ("cnt", "idx", "selected"):
        assert np.array_equal(ma[k], mb[k]), k
    assert ra["n_eff"] == rb["n_eff"] and np.array_equal(ra["HTH"], rb["HTH"])


# ------------------------------------------------------------------ 2. the sharded NDT target, voxel by voxel
def _ndt_target(tile):
    """The centred block at 0.25 m plus a dense column pair astride the negative tile edge x = y = -tile (NDT voxels of 1 m:
    voxel c spans [c + 0.5, c + 1.5), so the columns sit in voxels -tile - 1 and -tile, in different tiles)."""
    from lsdreg import synth
    m = synth.block_map(1, 1, 1, 0.25)
    m[:, :2] -= SHIFT[:2].astype(np.float32)
    rng = np.random.default_rng(5)
    cols = []
    for cx in (-tile - 1, -tile):
        for cy in (-tile - 1, -tile):
            p = rng.uniform(-0.45, 0.45, (40, 3)) + [cx + 1.0, cy + 1.0, 0.0]
            p[:, 2] = rng.uniform(0.6, 4.4, 40)
            cols.append(p)
    c = np.concatenate(cols)
    return np.concatenate([m, np.concatenate([c, np.zeros((len(c), 1))], 1).astype(np.float32)])


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("tile", [8, 3])
def test_sharded_ndt_target_voxel_by_voxel(world, tile):
    import lsdreg
    from lsdreg import shard
    m = _ndt_target(tile)
    single = lsdreg.Matcher("NDT_CUDA")
    single.set_target(m)
    full = single.voxels()
    key = {tuple(c): i for i, c in enumerate(full["coord"].tolist())}
    assert len(key) == len(full["count"])
    for cx in (-tile - 1, -tile):
        for z in range(1, 4):
            assert (cx, cx, z) in key or (cx, cx, z - 1) in key
    own = shard.tile_owner(full["coord"][:, 0], full["coord"][:, 1], tile, world)
    ranks = [lsdreg.Matcher("NDT_CUDA") for _ in range(world)]
    blobs = np.stack([r.shard_export(k, world, tile) for k, r in enumerate(ranks)])
    for r in ranks:
        r.shard_connect(blobs)
    _run_threads([lambda r=r: r.set_target(m) for r in ranks])
    seen = np.zeros(len(key), int)
    exact = True
    for k, r in enumerate(ranks):
        v = r.voxels()
        idx = np.array([key.get(tuple(c), -1) for c in v["coord"].tolist()])
        assert (idx >= 0).all(), f"rank {k}: voxels not in the unsharded table: {v['coord'][idx < 0][:4]}"
        assert len(np.unique(idx)) == len(idx)
        assert np.array_equal(np.sort(idx), np.nonzero(own == k)[0]), f"rank {k} of {world}: not exactly its tiles' voxels"
        seen[idx] += 1
        assert np.array_equal(v["count"], full["count"][idx])
        for f in ("mean", "second"):
            a, b = v[f], full[f][idx]
            assert np.all(np.abs(a - b) <= 1e-13 * np.abs(b).max(1, keepdims=True)), (k, f)
            exact &= np.array_equal(a, b)
        assert r.stats()["n_voxels"] == len(idx)
    assert (seen == 1).all()                                  # the union is the whole table, no voxel twice
    print(f"NDT world {world} tile {tile}: {len(key)} voxels, moments bit-identical: {exact}")
