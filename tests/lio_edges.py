"""TEST INFRASTRUCTURE: a map and two scans that put LIO scan points on the edges of h_share_model_geometric's per-point
logic (laserMapping.cpp:813-982) and of map_incremental (laserMapping.cpp:523-576), for tests/test_gpu_lio_edges.py (the
device against the compiled reference) and tests/test_lio_edges_host.py (the compiled reference reaches every class).

The pose and the extrinsic are the identity, so a scan point's world coordinates are its body coordinates, bit for bit.
Every item lives in its own region, at least 2 m from any other, so that its neighbour search (NEARBY18 at 0.5 m) sees
only its own map points.  Scan 1 items, by label:

  few_1 .. few_4  1 to 4 map points in range: a row with fewer than 5 neighbours (not selected; map_incremental's box test
                  on near[0], then PointToAdd)
  empty           nothing in range: an empty row
  collinear       6 map points exactly on a line (dyadic coordinates): esti_plane's QR of rank 2
  duplicate       6 copies of one map point: rank 1
  origin_plane    a plane through the world origin close to the sensor (A n = -1 has no solution), scan points on it
  body_zero       scan points at body (0, 0, 0) and (-0, 0, -0) on that plane: s = 1 - 0.9 |pd2| / sqrt(0)
  s_next, s_at_above, s_at_below, s_prev
                  a horizontal plane of 5 points and a scan point above it, placed (tune_gate) so that the fp32 s of
                  laserMapping.cpp:861 is the float after 0.9f (kept), 0.9f with the double s above 0.9f (dropped; kept
                  by `s > 0.9f`), 0.9f with the double s at or below it, and the float before 0.9f
  plane           tilted planes with noise: the ordinary selected point
  fsize_pos, fsize_neg, fsize_negzero
                  world coordinates on multiples of filter_size_map_min = 0.5 (positive, negative, -0.0) in a dense patch
  box_tie_1, box_tie_2, box_tie_3
                  one neighbour exactly 0.5 fsize from the downsample box centre on 1, 2 or 3 axes and more than that
                  on the others: the strict `>` keeps it out of PointNoNeedDownsample
  box_out         one neighbour beyond 0.5 fsize on all three axes: PointNoNeedDownsample
  dist_tie        5 neighbours, two of them exactly as far from the box centre as the point (calc_dist ties), the
                  others farther: PointToAdd (`<` is strict)
  dist_less       the same with one neighbour nearer than the point: not added
  stale_keep, stale_drop
                  scan 2 moves these points of a horizontal plane 200 m along it (stale_keep: the stale row still
                  fits) or 200 m along every axis (stale_drop: its near[0] is then beyond the box on all three, so
                  PointNoNeedDownsample); the search finds nothing there and the row of scan 1 is kept

Scan 2 is scan 1 with the stale_* points moved.  Both scans have the same size, so every row carries over."""
import numpy as np

FSIZE = 0.5
F32 = np.float32
NEXT_09 = np.nextafter(F32(0.9), F32(1.0))
PREV_09 = np.nextafter(F32(0.9), F32(0.0))


def s_gate(pabcd, world, body):
    """laserMapping.cpp:860-862 as the reference evaluates it: pd2 in fp32 left to right, s in double, the gate on the fp32 s
    against the double 0.9.  -> (pd2 float32, s float64, s float32, kept)."""
    a = np.asarray(pabcd, F32); w = np.asarray(world, F32)
    pd2 = ((a[..., 0] * w[..., 0] + a[..., 1] * w[..., 1]) + a[..., 2] * w[..., 2]) + a[..., 3]
    b = np.asarray(body, F32)[..., :3].astype(np.float64)
    nrm = np.sqrt((b[..., 0] * b[..., 0] + b[..., 1] * b[..., 1]) + b[..., 2] * b[..., 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        s = 1 - 0.9 * np.abs(pd2.astype(np.float64)) / np.sqrt(nrm)
    sf = s.astype(F32)
    return pd2, s, sf, sf.astype(np.float64) > 0.9


def s_class(s, sf):
    """The gate class of points whose plane fitted: an array of s_* labels, "" where none applies."""
    s, sf = np.asarray(s), np.asarray(sf)
    at = sf == F32(0.9)
    return np.select([sf == NEXT_09, at & (s > float(F32(0.9))), at, sf == PREV_09],
                     ["s_next", "s_at_above", "s_at_below", "s_prev"], "")


class Scene:
    def __init__(self):
        self.map = []
        self.scan = []
        self.label = []

    def m(self, pts):
        self.map.append(np.asarray(pts, F32).reshape(-1, 3))

    def s(self, pts, label):
        p = np.asarray(pts, F32).reshape(-1, 3)
        self.scan.append(p)
        self.label += [label] * len(p)

    def arrays(self):
        m = np.concatenate(self.map)
        mp = np.zeros((len(m), 4), F32); mp[:, :3] = m
        s = np.concatenate(self.scan)
        sp = np.zeros((len(s), 4), F32); sp[:, :3] = s
        return mp, sp, np.array(self.label)


def _far_region(k):
    """Centre of the k-th isolated region: voxel-aligned (multiples of 0.5), 3 m apart, 10 to 40 m from the sensor."""
    return np.array([10.0 + 3.0 * (k % 10), 10.0 + 3.0 * (k // 10), 1.0])


# the gate regions: voxel centres 2.5 to 4.5 m from the sensor, so that the point sits at h = 0.11 sqrt(|p|) < 0.25 m above
# its plane, inside the voxel of its 5 neighbours
S_CENTRES = [(-3.5, -2.5), (-1.5, -3.0), (1.5, -3.0), (3.5, -2.5), (-3.5, 2.5), (-1.5, 3.0), (1.5, 3.0), (3.5, 2.5),
             (-3.5, 0.0), (3.5, 0.0), (0.0, -4.0), (0.0, 4.0)]
S_Z0 = -1.0
S_LABELS = ["s_next", "s_at_above", "s_at_below", "s_prev"]


def build(rng=None, gate=None):
    """-> dict(map [m,4], scan1 [n,4], scan2 [n,4], label [n]).  gate: {scan index: position} from tune_gate; without it the
    gate points sit at their first guess."""
    rng = np.random.default_rng(5) if rng is None else rng
    sc = Scene()
    k = 0

    def region():
        nonlocal k
        c = _far_region(k); k += 1
        return c

    for cnt in (1, 2, 3, 4):
        for _ in range(4):
            c = region()
            sc.m(c + rng.uniform(-0.2, 0.2, (cnt, 3)))
            sc.s(c + rng.uniform(-0.1, 0.1, 3), f"few_{cnt}")
    for _ in range(4):
        sc.s(region(), "empty")
    for _ in range(4):
        c = region()
        d = np.array([1.0, 0.5, 0.25]) * rng.choice([-1, 1], 3)
        sc.m(c + np.array([-0.1875, -0.125, -0.0625, 0.0625, 0.125, 0.1875])[:, None] * d)
        sc.s(c + np.array([0.0, 0.0625, 0.0625]), "collinear")
    for _ in range(4):
        c = region()
        sc.m(np.repeat([c + np.array([0.0625, 0.125, 0.0])], 6, 0))
        sc.s(c + np.array([0.0, 0.0, 0.0625]), "duplicate")
    # a plane through the origin, normal (1, 2, -3)
    n = np.array([1.0, 2.0, -3.0]) / np.sqrt(14.0)
    e1 = np.cross(n, [1.0, 0, 0]); e1 /= np.linalg.norm(e1)
    e2 = np.cross(n, e1)
    uv = rng.uniform(-0.6, 0.6, (80, 2))
    sc.m(uv[:, :1] * e1 + uv[:, 1:] * e2)
    uv = rng.uniform(-0.4, 0.4, (10, 2))
    sc.s(uv[:, :1] * e1 + uv[:, 1:] * e2 + n * rng.normal(0, 0.005, (10, 1)), "origin_plane")
    sc.s([[0.0, 0.0, 0.0], [-0.0, 0.0, -0.0]], "body_zero")
    # the gate: 5 neighbours on z = S_Z0 around a voxel centre, the scan point above it
    for j, (x, y) in enumerate(S_CENTRES):
        c = np.array([x, y, S_Z0])
        sc.m(c + np.c_[np.array([[-0.1875, -0.125], [0.1875, -0.0625], [0.0, 0.1875], [-0.125, 0.125], [0.125, 0.0625]]), np.zeros(5)])
        p = np.array([x, y, S_Z0])
        for _ in range(20):                     # s = 0.9 <=> h = 0.1 / 0.9 sqrt(|p|), p = (x, y, S_Z0 + h)
            p[2] = S_Z0 + np.sqrt(np.linalg.norm(p)) * 0.1 / 0.9
        sc.s(p, S_LABELS[j % 4])
    # ordinary tilted planes
    for _ in range(8):
        c = region()
        nn = rng.normal(size=3); nn[2] += 3; nn /= np.linalg.norm(nn)
        a = np.cross(nn, [1.0, 0, 0]); a /= np.linalg.norm(a); b = np.cross(nn, a)
        uv = rng.uniform(-0.7, 0.7, (40, 2))
        sc.m(c + uv[:, :1] * a + uv[:, 1:] * b + nn * rng.normal(0, 0.01, (40, 1)))
        uv = rng.uniform(-0.3, 0.3, (4, 2))
        sc.s(c + uv[:, :1] * a + uv[:, 1:] * b + nn * rng.normal(0, 0.01, (4, 1)), "plane")
    # world points on multiples of fsize, in dense horizontal patches (z = 0.5 m steps as well)
    for c, lab in (((20.0, -12.0, 1.5), "fsize_pos"), ((-10.0, -12.0, -2.0), "fsize_neg"), ((0.0, -16.0, 1.0), "fsize_negzero")):
        c = np.array(c)
        sc.m(c + np.c_[rng.uniform(-1.2, 1.2, (120, 2)), rng.normal(0, 0.02, 120)])
        g = c + np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [-0.5, 0.5, 0.0], [1.0, -0.5, 0.0], [0.0, 0.0, 0.5], [-1.0, 1.0, 0.0]])
        if lab == "fsize_negzero":
            g[:, 0] = -0.0 * np.ones(len(g)); g[4:, 0] = [-0.0, 0.0]
        sc.s(g, lab)
    # map_incremental's box test: one neighbour at mid + offset (exact in fp32), the point near the box centre
    for lab, off in (("box_tie_1", (0.25, 0.375, -0.375)), ("box_tie_2", (-0.25, 0.25, 0.375)), ("box_tie_3", (0.25, -0.25, 0.25)),
                     ("box_out", (0.375, 0.375, -0.375))):
        for _ in range(3):
            mid = region() + 0.25
            sc.m(mid + np.array(off))
            sc.s(mid + np.array([0.0625, -0.0625, 0.0]), lab)
    # calc_dist ties: w = mid + (a, b, c), two neighbours mirrored through mid (the same squared distance, exactly), three
    # farther from mid; dist_less moves one of those three nearer than w
    for lab in ("dist_tie", "dist_less"):
        for _ in range(3):
            mid = region() + 0.25
            w = np.array([0.125, 0.0625, 0.1875])
            q = [w * [-1, 1, 1], w * [1, -1, -1], [0.25 - 1 / 64, 0.0, 0.1875], [0.0, 0.25 - 1 / 64, -0.1875], [-0.1875, -0.1875, 0.0]]
            if lab == "dist_less":
                q[4] = [0.0625, 0.0625, 0.0625]
            sc.m(mid + np.array(q))
            sc.s(mid + w, lab)
    # stale rows: points of a horizontal plane at z = 1.0, moved in scan 2
    stale_src = []
    for lab in ("stale_keep", "stale_drop"):
        c = region()
        c[2] = 1.0
        sc.m(c + np.c_[rng.uniform(-0.7, 0.7, (40, 2)), np.zeros(40)])
        sc.s(c + np.c_[rng.uniform(-0.3, 0.3, (4, 2)), np.zeros(4)], lab)
    mp, s1, label = sc.arrays()
    if gate:
        for i, p in gate.items():
            s1[i, :3] = p
    s2 = s1.copy()
    keep, drop = label == "stale_keep", label == "stale_drop"
    s2[keep, :2] += F32(200.0)
    s2[drop, :3] += F32(200.0)
    return dict(map=mp, scan1=s1, scan2=s2, label=label)


def _ord(f):
    b = np.asarray(f, F32).view(np.int32).astype(np.int64)
    return np.where(b >= 0, b, -(b & 0x7FFFFFFF))


def _unord(o):
    o = np.asarray(o, np.int64)
    return np.where(o >= 0, o, (-o) | 0x80000000).astype(np.uint32).view(F32)


def tune_gate(rows, scene, span=300):
    """Place every s_* point so that the gate lands in its class.  rows [n,5,3]: the neighbour rows the compiled reference
    returned for the first-guess scene (in its order: for 5 candidates the order they are gathered in, which a move of a
    few ulps does not change).  The plane is the compiled esti_plane's fit of that row; the point's x and z are walked over
    +-span fp32 values and the nearest position of the wanted class taken.  -> {scan index: xyz}."""
    from oracle import oracle as O
    out = {}
    lab = scene["label"]
    idx = np.nonzero(np.char.startswith(lab.astype(str), "s_"))[0]
    pabcd, ok = O.ref_esti_plane(rows[idx], 0.1)
    steps = np.arange(-span, span + 1)
    for t, i in enumerate(idx):
        assert ok[t] == 1, "a gate plane was rejected"
        p0 = scene["scan1"][i, :3]
        xs = _unord(_ord(p0[0]) + steps)
        zs = _unord(_ord(p0[2]) + steps)
        X, Z = np.meshgrid(xs, zs, indexing="ij")
        w = np.stack([X, np.full_like(X, p0[1]), Z], -1)
        _, s, sf, _ = s_gate(pabcd[t], w, w)
        want = lab[i]
        hit = s_class(s, sf) == want
        assert hit.any(), f"no position of class {want} within +-{span} fp32 steps of point {i}"
        d = np.abs(steps)[:, None] + np.abs(steps)[None, :]
        a, b = np.unravel_index(np.where(hit, d, 1 << 30).argmin(), d.shape)
        out[int(i)] = w[a, b]
    return out


# ---------------------------------------------------------------- the compiled reference's side
def identity_state():
    from oracle import eskf
    return eskf.State().to_vec()


def make_oracle(scene, reference_order):
    """OracleLio on the scene's map: with reference_order the compiled iVox, esti_plane and map_incremental
    (oracle/_ref/libref_lio.so, ref_lio_hmodel / ref_map_incremental); without it the port, whose rows are in ascending
    (d2, id) order as the device's then are (its esti_plane is pinned bit for bit to Eigen's by tests/test_oracle_golden.py).
    Rows outlive a search that finds nothing (stale_neighbours), as laserMapping.cpp's Nearest_Points do."""
    from oracle.lio import OracleLio
    o = OracleLio(18, expected_cells=1 << 14, stale_neighbours=True, reference_order=reference_order, degenerate_detect=False,
                  backend="reference" if reference_order else "port", nthreads=1)
    o.add_map_points(scene["map"])
    n = len(scene["scan1"])
    o.near_xyz = np.zeros((n, 5, 3), F32); o.near_ids = np.full((n, 5), -1, np.int32)
    o.near_cnt = np.zeros(n, np.int32); o.selected = np.ones(n, np.uint8)
    return o


def oracle_eval(o, body, search):
    """One h_share_model_geometric evaluation at the identity pose -> the per-point taps and the Jacobian rows."""
    from oracle import eskf
    n = len(body)
    o.world = np.zeros((n, 4), F32); o.plane = np.zeros((n, 4), F32)
    r = o._hmodel(np.ascontiguousarray(body, F32), eskf.State(), search)
    return dict(world=o.world.copy(), cnt=o.near_cnt[:n].copy(), idx=o.near_ids[:n].copy(), xyz=o.near_xyz[:n].copy(),
                selected=o.selected[:n].copy(), plane=o.plane.copy(), h_x=r["h_x"][:, :6].copy(), h=r["h"].copy(),
                n_eff=r["n"], res_sum=o.last["res_sum"])


def oracle_map_incremental(o, body, ekf_inited):
    from oracle import eskf
    o.x = eskf.State()
    o.ekf_inited = bool(ekf_inited)
    id0 = o.next_id
    o.map_incremental(np.ascontiguousarray(body, F32))
    return dict(flags=o.flags.copy(), world=o.world.copy(), id0=id0)


def tuned_scene(reference_order):
    """The scene with its gate points placed against the rows this oracle's search returns."""
    s0 = build()
    o = make_oracle(s0, reference_order)
    r = oracle_eval(o, s0["scan1"], True)
    return build(gate=tune_gate(r["xyz"], s0))


def classes(scene, ev, mi=None):
    """Per-class counts of one evaluation (and the map_incremental after it), read off the oracle's own outputs."""
    from oracle import oracle as O
    lab = scene["label"]
    cnt, sel = ev["cnt"], ev["selected"].astype(bool)
    out = {f"cnt_{k}": int((cnt == k).sum()) for k in range(5)}
    out["cnt_5"] = int((cnt == 5).sum())
    full = cnt >= 5
    nz = np.zeros(len(lab), np.int32)
    if full.any():
        nz[full] = O.ref_esti_plane_qr(ev["xyz"][full])["nonzero_pivots"] if O.HAVE_REF else O.esti_plane_qr(ev["xyz"][full])["nonzero_pivots"]
    out["rank_2_row"] = int((full & (nz == 2)).sum())
    out["rank_1_row"] = int((full & (nz == 1)).sum())
    out["origin_plane_fit"] = int((full & (lab == "origin_plane")).sum())
    out["body_zero_fit"] = int((full & (lab == "body_zero")).sum())
    out["selected"] = int(sel.sum())
    out["not_selected_with_row"] = int((full & ~sel).sum())
    # the gate classes: the plane the oracle fits to its own row, the point where the oracle put it
    pl, ok = (O.ref_esti_plane if O.HAVE_REF else O.esti_plane)(ev["xyz"], 0.1)
    _, s, sf, kept = s_gate(pl, ev["world"][:, :3], ev["world"][:, :3])
    cls = s_class(s, sf)
    for c in S_LABELS:
        m = full & (ok == 1) & (cls == c)
        out[c] = int(m.sum())
        assert (sel[m] == (c == "s_next")).all(), c
    if mi is not None:
        f = mi["flags"]
        for v in (0, 1, 2):
            out[f"flag_{v}"] = int((f == v).sum())
        for c in ("box_tie_1", "box_tie_2", "box_tie_3"):
            out[c] = int(((lab == c) & (cnt == 1) & (f == 1)).sum())
        out["box_out"] = int(((lab == "box_out") & (cnt == 1) & (f == 2)).sum())
        out["dist_tie"] = int(((lab == "dist_tie") & full & (f == 1)).sum())
        out["dist_less"] = int(((lab == "dist_less") & full & (f == 0)).sum())
        for c in ("fsize_pos", "fsize_neg", "fsize_negzero"):
            out[c] = int(((lab == c) & (cnt > 0)).sum())
        out["fewer_than_5"] = int(((cnt > 0) & (cnt < 5) & (f == 1)).sum())
    return out


def stale_classes(scene, ev2, mi2):
    """Scan 2: rows kept from scan 1 because the search found nothing."""
    lab = scene["label"]
    st = np.isin(lab, ["stale_keep", "stale_drop"]) & (ev2["cnt"] >= 5)
    return dict(stale_row=int(st.sum()), stale_selected=int((st & (ev2["selected"] == 1)).sum()),
                stale_no_need_downsample=int((st & (mi2["flags"] == 2)).sum()), stale_to_add=int((st & (mi2["flags"] == 1)).sum()))
