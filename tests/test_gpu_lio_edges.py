"""GPU parity of the LIO scan step's per-point logic at its edges, against the compiled reference (oracle/_ref) point by
point:
  * esti_plane_dev alone (lsd_debug_esti_plane) on the committed sets of tests/golden/esti_plane_edges.npz, whose answers
    are Eigen's ColPivHouseholderQR compiled from the reference (tests/golden/make_golden_esti_plane.py), and, where the
    compiled reference is present, on the same families drawn at about 10^5 sets;
  * linearize (search, then the cached-plane reuse path) and map_incremental on the scene of tests/lio_edges.py: world
    bits, neighbour counts, ids and coordinates, selected flags, plane bits, map_incremental flags and the map's contents,
    for both neighbour orders.
Every edge class of the scene is counted on the reference's own outputs and must be non-empty."""
import importlib.util
import math
import os
from collections import Counter

import numpy as np
import pytest

import lio_edges as L
from oracle import oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "esti_plane_edges.npz")


def _same_bits(a, b):
    """Bit for bit, any NaN equal to any NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _check_planes(pts, pabcd, ok, what):
    import lsdreg
    gp, gok = lsdreg.capi.debug_esti_plane(pts, 0.1)
    bad = ~_same_bits(gp, pabcd).all(1) | (gok != ok)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {len(pts)} sets differ, first {np.nonzero(bad)[0][:8]}: {gp[bad][:2]} vs {pabcd[bad][:2]}"


def test_esti_plane_on_the_device_is_eigens():
    g = np.load(GOLD)
    pts, nz, perm = g["pts"], g["nz"].astype(int), g["perm"].astype(int)
    # classes by Eigen's own factorisation: non-zero pivots and column permutation.  Eigen never reports 0 non-zero pivots:
    # at k = 0 its test compares the largest column norm with itself times epsilon; the all-zero sets are the class that
    # stands for it (3 "non-zero" pivots of value 0, a NaN plane).
    cls = Counter(zip(nz.tolist(), map(tuple, perm.tolist())))
    print("esti_plane classes (non-zero pivots, permutation):", dict(sorted(cls.items())))
    fam = g["families"][g["family"]]
    print("families:", dict(Counter(fam.tolist())))
    for k in (1, 2, 3):
        for p in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
            assert cls[(k, p)] > 0, (k, p)
    assert (np.isnan(g["pabcd"]).any(1) & (np.abs(pts) == 0).all((1, 2))).sum() >= 40
    thr = fam == "threshold"
    assert (g["ok"][thr] == 1).sum() > 200 and (g["ok"][thr] == 0).sum() > 200
    _check_planes(pts, g["pabcd"], g["ok"], "committed sets")
    if O.HAVE_REF and hasattr(O.ref, "ref_esti_plane_qr"):
        spec = importlib.util.spec_from_file_location("make_golden_esti_plane", os.path.join(HERE, "golden", "make_golden_esti_plane.py"))
        gen = importlib.util.module_from_spec(spec); spec.loader.exec_module(gen)
        big, _, _ = gen.edge_sets(O, np.random.default_rng(7), scale=4.0)          # about 1.3 10^5 sets
        rp, rok = O.ref_esti_plane(big, 0.1)
        print(f"{len(big)} further sets against the compiled reference")
        _check_planes(big, rp, rok, "sets drawn against the compiled reference")


# ---------------------------------------------------------------- the scene
def _frontend(scene, reference_order, reuse):
    import lsdreg
    if reuse == "cluster":
        os.environ["LSD_REUSE_CLUSTER"] = "8x1024"
    try:
        g = lsdreg.LioFrontend(map_log2_lines=14, degenerate_detect_en=0, max_points=4096)
    finally:
        os.environ.pop("LSD_REUSE_CLUSTER", None)
    g.set_reference_order(reference_order)
    g.map.insert(scene["map"], 0)
    g.set_next_id(scene["map"].shape[0])
    return g


def _compare_eval(g, rg, ev, what):
    mt = g.get_matches()
    n = len(ev["cnt"])
    assert (mt["world"][:, :3].view(np.uint32) == ev["world"][:, :3].view(np.uint32)).all(), what
    bad = np.nonzero(mt["cnt"] != ev["cnt"])[0]
    assert not len(bad), f"{what}: cnt differs at {bad[:8]}: {mt['cnt'][bad[:8]]} vs {ev['cnt'][bad[:8]]}"
    bad = np.nonzero((mt["idx"] != ev["idx"]).any(1))[0]
    assert not len(bad), f"{what}: ids differ at {bad[:8]}"
    assert (mt["xyz"].view(np.uint32) == ev["xyz"].view(np.uint32)).all(), what
    bad = np.nonzero(mt["selected"] != ev["selected"])[0]
    assert not len(bad), f"{what}: selected differs at {bad[:8]}: {mt['selected'][bad[:8]]} vs {ev['selected'][bad[:8]]}"
    sel = mt["selected"].astype(bool)
    bad = np.nonzero(~_same_bits(mt["plane"][sel], ev["plane"][sel]).all(1))[0]
    assert not len(bad), f"{what}: plane bits differ at {np.nonzero(sel)[0][bad[:8]]}"
    assert rg["n_eff"] == ev["n_eff"] == int(sel.sum()), what
    # HTH and HTh against exact sums of the reference's rows.  Each term is one double product, formed identically on
    # both sides (at the identity pose the device's row equals the reference's h_x row).  The device adds the n_eff
    # products in some order; recursive summation of m terms in any order is within gamma_(m-1) * sum|terms| of the exact
    # sum, gamma_k = k u / (1 - k u), u = 2^-53.  For m <= 2^40, gamma_(m-1) < m 2^-52, the bar below.
    hx, h = ev["h_x"], ev["h"]
    m = len(h)
    for a in range(6):
        for c in range(6):
            t = hx[:, a] * hx[:, c]
            assert abs(rg["HTH"][a, c] - math.fsum(t)) <= m * 2.0 ** -52 * math.fsum(np.abs(t)), (what, a, c)
        t = hx[:, a] * h
        assert abs(rg["HTh"][a] - math.fsum(t)) <= m * 2.0 ** -52 * math.fsum(np.abs(t)), (what, a)
    t = np.abs(h)
    assert abs(rg["res_sum"] - math.fsum(t)) <= m * 2.0 ** -52 * math.fsum(t), what


def _map_mirror(scene):
    """The compiled iVox holding the scene's map, fed each map_incremental's two AddPoints calls (laserMapping.cpp:571-572)."""
    r = O.RefIvox(0.5, 18)
    r.add(scene["map"], 0)
    return r


def _compare_map_incremental(g, r, mi, id_t2, what):
    from test_gpu_map_contents import assert_same, device_contents, ref_contents
    flags, _ = g.get_map_flags()
    bad = np.nonzero(flags != mi["flags"])[0]
    assert not len(bad), f"{what}: map_incremental flags differ at {bad[:8]}: {flags[bad[:8]]} vs {mi['flags'][bad[:8]]}"
    world = g.get_matches()["world"]
    assert (world[:, :3].view(np.uint32) == mi["world"][:, :3].view(np.uint32)).all(), what
    if r is not None:            # port oracle: the compiled iVox mirrors the map from the (equal) flags
        i = np.arange(len(flags))
        for f in (1, 2):
            s = flags == f
            r.add_ids(world[s], (mi["id0"] + i[s] + (id_t2 if f == 2 else 0)).astype(np.int32))
    return device_contents(g.map)


@pytest.mark.skipif(not O.HAVE_REF_IVOX_DUMP, reason="oracle/_ref/libref_lio.so not built (needs the reference tree)")
@pytest.mark.parametrize("reference_order,reuse,ekf_inited", [(True, "grid", True), (True, "cluster", True), (False, "grid", True),
                                                               (False, "cluster", True), (True, "grid", False)])
def test_lio_edges_match_compiled_reference(reference_order, reuse, ekf_inited):
    from test_gpu_map_contents import assert_same, ref_contents
    if reuse == "cluster" and os.environ.get("LSDREG_EMU"):
        pytest.skip("thread-block clusters do not exist under the SIMT emulator")
    scene = L.tuned_scene(reference_order)
    g = _frontend(scene, reference_order, reuse)
    g.set_ekf_inited(ekf_inited)
    o = L.make_oracle(scene, reference_order)
    mirror = None if reference_order else _map_mirror(scene)
    x = L.identity_state()
    counts = Counter()
    for k, body in enumerate((scene["scan1"], scene["scan2"])):
        n = g.load_scan(body, downsample=False)
        assert n == len(body)
        ev = L.oracle_eval(o, body, True)
        _compare_eval(g, g.linearize(x, True), ev, f"scan {k} search")
        ev_reuse = L.oracle_eval(o, body, False)
        _compare_eval(g, g.linearize(x, False), ev_reuse, f"scan {k} reuse")
        mi = L.oracle_map_incremental(o, body, ekf_inited)
        added = g.map_incremental(x)
        assert added == int((mi["flags"] > 0).sum())
        id_t2 = n if reference_order else 0
        dev = _compare_map_incremental(g, mirror, mi, id_t2, f"scan {k}")
        ref = ref_contents(o.map if reference_order else mirror)
        assert_same(dev, ref, reference_order, f"scan {k}: compiled iVox")
        if k == 0:
            counts.update(L.classes(scene, ev, mi))
            counts.update({f"reuse_{c}": v for c, v in L.classes(scene, ev_reuse).items() if c.startswith("s_")})
        else:
            counts.update(L.stale_classes(scene, ev, mi))
    print("edge classes:", dict(counts))
    if ekf_inited:
        empty = [c for c, v in counts.items() if v == 0]
        assert not empty, f"edge classes the scene failed to reach: {empty}"
    else:
        assert counts["flag_1"] == len(scene["scan1"])          # flg_EKF_inited == 0: every point is PointToAdd


@pytest.mark.skipif(not O.HAVE_REF_IVOX_DUMP, reason="oracle/_ref/libref_lio.so not built (needs the reference tree)")
@pytest.mark.parametrize("reference_order", [True, False])
def test_seeding_scan_matches_compiled_reference(reference_order):
    """The first scan on an empty map (laserMapping.cpp:1227-1239): every point added, ids id0 + i, the same map."""
    import lsdreg
    from test_gpu_map_contents import assert_same, device_contents, ref_contents
    scene = L.build()
    g = lsdreg.LioFrontend(map_log2_lines=14, max_points=4096)
    g.set_reference_order(reference_order)
    g.set_next_id(77)
    P = lsdreg.init_cov()
    x1, _, info = g.scan(scene["map"], L.identity_state(), P)
    assert info["status"] == lsdreg.MAP_SEEDED
    flags, _ = g.get_map_flags()
    body = g.get_down()
    assert (flags == 1).all() and len(flags) == len(body) == info["n_added"]
    r = O.RefIvox(0.5, 18)
    r.add_ids(body, (77 + np.arange(len(body))).astype(np.int32))
    assert_same(device_contents(g.map), ref_contents(r), True, "seeded map")
