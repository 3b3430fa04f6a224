"""GPU: what the hash-voxel map holds, voxel by voxel (lsd_map_dump), against the compiled iVox (oracle/_ref, when built)
and against a restatement of IVox::AddPoints (ivox3d.h:232-256) that is itself pinned to the compiled iVox by the same
dumps.  Bars, after every operation:
  * the same set of voxel keys (the reference's keys come from Pos2Grid evaluated in C++: Eigen rounds half away from zero);
  * per voxel, the same multiset of (x, y, z, id) bit patterns, tombstones excluded;
  * stats() equals the dump's totals (cells = voxels in the table, points = live points);
  * where the ids are ascending in AddPoints order, the device's points sorted by id are the reference's insertion order
    of the voxel (what lsd_lio_set_reference_order rests on).
Every LRU case asserts, through the restatement's counters, that the path it is about was actually taken.
The map-level cases also run on the CPU under the SIMT emulator (tests/simt/fuzz_map_contents.py)."""
import os
from collections import Counter, OrderedDict, defaultdict

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EMU = bool(os.environ.get("LSDREG_EMU"))      # SIMT emulator build: x86 float -> int conversions, small workloads


# ------------------------------------------------------------------ restatement of IVox::AddPoints
class IvoxRestated:
    """IVox::AddPoints (ivox3d.h:232-256): grids_cache_ as an OrderedDict whose LAST entry is the list's front.  Each voxel
    holds its points in insertion order as (x bits, y bits, z bits, id).  Counters record the LRU paths a batch took."""

    def __init__(self, res: float, capacity=None, max_distance: float = 100.0):
        self.inv = np.float32(1.0 / np.float64(np.float32(res)))        # options_.inv_resolution_ = 1.0 / resolution_
        self.cap = (1 << 62) if capacity is None else int(capacity)
        self.maxd = float(max_distance)
        self.grid = OrderedDict()                                       # key -> [creation distance, [points]]
        self.n = Counter()
        self._open = None                                               # (evictions, points per voxel) of the batch in progress

    def keys(self, xyz):
        """Pos2Grid: (p * inv_resolution_).round() in float, half away from zero."""
        v = (np.asarray(xyz, np.float32)[:, :3] * self.inv).astype(np.float64)
        a = np.abs(v)
        r = np.floor(a)
        r += (a - r) >= 0.5
        return (np.sign(v) * r).astype(np.int64)

    def add(self, xyz, ids, distance: float, batch_end: bool = True):
        """One AddPoints call.  The counters describe the product's batch, which may span several calls (map_incremental
        replays a scan's two calls as one batch): batch_end=False carries the batch on into the next call."""
        xyz = np.ascontiguousarray(np.asarray(xyz, np.float32)[:, :3])
        if self._open is None:
            self._open = (Counter(), defaultdict(list))
        evicted, gone = self._open                                      # gone: ids of the points each eviction dropped
        for k, b, i in zip(map(tuple, self.keys(xyz).tolist()), xyz.view(np.uint32).tolist(), np.asarray(ids).tolist()):
            c = self.grid.get(k)
            if c is None:
                c = self.grid[k] = [distance, []]
            else:
                self.grid.move_to_end(k)
            c[1].append((*b, i))
            if len(self.grid) > self.cap:
                back = next(iter(self.grid))
                if distance - self.grid[back][0] > self.maxd:
                    gone[back] += [t[3] for t in self.grid.pop(back)[1]]
                    evicted[back] += 1
        if not batch_end:
            return
        self._open = None
        self.n["evicted"] += sum(evicted.values())
        for k, m in evicted.items():
            self.n["evicted_twice"] += m >= 2
            if k not in self.grid:
                continue
            surv = [t[3] for t in self.grid[k][1]]
            self.n["recreated"] += 1
            self.n["recreated_over_8"] += len(surv) > 8
            self.n["max_survivors"] = max(self.n["max_survivors"], len(surv))
            # keeping "ids >= the re-creating point's id" among everything the voxel held would keep a different set: ids
            # not monotone in AddPoints order (or an id wrap)
            self.n["order_breaks"] += {i for i in gone[k] + surv if i >= surv[0]} != set(surv)

    def delete_boxes(self, boxes):
        """KD_TREE::Delete_Point_Boxes on the voxels' points: deleted iff min <= p < max on every axis, for any box."""
        b = np.asarray(boxes, np.float32).reshape(-1, 6)
        n = 0
        for c in self.grid.values():
            keep = []
            for t in c[1]:
                p = np.array(t[:3], np.uint32).view(np.float32)
                if ((b[:, :3] <= p) & (b[:, 3:] > p)).all(axis=1).any():
                    n += 1
                else:
                    keep.append(t)
            c[1] = keep
        return n

    def contents(self):
        return {k: list(c[1]) for k, c in self.grid.items() if c[1]}


# ------------------------------------------------------------------ read-backs and comparison
def device_contents(g):
    """Live points per voxel in storage order; asserts stats() against the dump's totals."""
    d = g.dump()
    st = g.stats()
    live = ~d["tombstone"]
    vox = [tuple(v) for v in d["voxel"].tolist()]
    assert st["cells"] == len(set(vox)) and st["points"] == int(live.sum()), (st, len(set(vox)), int(live.sum()))
    out = {}
    bits = np.ascontiguousarray(d["xyz"]).view(np.uint32).tolist()
    for v, b, i, alive in zip(vox, bits, d["id"].tolist(), live.tolist()):
        if alive:
            out.setdefault(v, []).append((*b, i))
    return out


def ref_contents(r):
    keys, xyz, ids = r.dump()
    out = {}
    for k, b, i in zip(map(tuple, keys.tolist()), np.ascontiguousarray(xyz).view(np.uint32).tolist(), ids.tolist()):
        out.setdefault(k, []).append((*b, i))
    return out


def assert_same(dev, ref, id_order: bool, what: str):
    if dev.keys() != ref.keys():
        a, b = set(dev) - set(ref), set(ref) - set(dev)
        raise AssertionError(f"{what}: voxel sets differ: {len(a)} only on the device {sorted(a)[:4]}, {len(b)} only in the reference {sorted(b)[:4]}")
    for k, pts in ref.items():
        dp = dev[k]
        assert sorted(dp) == sorted(pts), f"{what}: voxel {k}: {len(dp)} points on the device, {len(pts)} in the reference; ids {sorted(t[3] for t in dp)[:12]} vs {sorted(t[3] for t in pts)[:12]}"
        if id_order:
            assert sorted(dp, key=lambda t: t[3]) == pts, f"{what}: voxel {k}: the device's points sorted by id are not the insertion order"


class Rig:
    """The device map, the restatement and (when built) the compiled iVox, fed the same AddPoints batches."""

    def __init__(self, res=0.5, log2_lines=14, capacity=None, max_distance=100.0, compiled=True):
        import lsdreg
        from oracle import oracle as O
        self.g = lsdreg.HashVoxelMap(res, log2_lines)
        if capacity is not None:
            self.g.enable_lru(capacity, max_distance)
        self.m = IvoxRestated(res, capacity, max_distance)
        self.r = O.RefIvox(res, 18, (1 << 30) if capacity is None else capacity, max_distance) if compiled and O.HAVE_REF_IVOX_DUMP else None
        self.next_id = 0
        self.deleted = False

    def add(self, xyz, distance=0.0, check=True):
        xyz = np.asarray(xyz, np.float32)
        n = xyz.shape[0]
        pts = np.zeros((n, 4), np.float32)
        pts[:, :3] = xyz[:, :3]
        ids = self.next_id + np.arange(n, dtype=np.int64)
        self.g.set_travel_distance(distance)
        self.g.insert(pts, self.next_id)
        self.m.add(pts, ids, distance)
        if self.r is not None:
            self.r.add_ids(pts, ids.astype(np.int32), distance)
        self.next_id += n
        if check:
            self.check()

    def delete_boxes(self, boxes):
        n = self.g.delete_boxes(boxes)
        assert n == self.m.delete_boxes(boxes)
        self.deleted = True          # the compiled iVox has no box delete: from here on the restatement is the reference
        self.check()
        return n

    def check(self):
        dev = device_contents(self.g)
        assert_same(dev, self.m.contents(), True, "restatement")
        if self.r is not None and not self.deleted:
            ref = ref_contents(self.r)
            assert_same(dev, ref, True, "compiled iVox")
            assert ref == self.m.contents(), "the restatement departs from the compiled iVox"
            assert self.r.num_cells == len(ref)
        return dev


def _cloud(rng, n, lo, hi):
    return rng.uniform(lo, hi, (n, 3)).astype(np.float32)


# ------------------------------------------------------------------ plain insert
def test_small_world_map_contents(small_world):
    rig = Rig(0.5, 19)
    rig.add(small_world["map"][:, :3])
    assert rig.g.stats()["dropped"] == 0


def test_crowded_voxel_negative_coordinates_and_half_boundaries():
    """One voxel through several overflow lines, points on both sides of zero, and points exactly on voxel half-boundaries
    (x * inv_res = k + 0.5, where half-away-from-zero and half-to-even part); ragged incremental insert == bulk insert."""
    rng = np.random.default_rng(11)
    crowd = np.array([-1.0, 2.0, -3.0], np.float32) + rng.uniform(-0.2, 0.2, (60, 3)).astype(np.float32)   # 60 points, 9 lines
    spread = _cloud(rng, 500, -6.0, 6.0)
    k = np.arange(-6, 7, dtype=np.float32)
    half = np.stack(np.meshgrid(k / 2 + 0.25, k[:5] / 2 + 0.25, np.float32([-0.75, 0.25, 0.75])), -1).reshape(-1, 3)
    assert ((half * 2) % 1 == 0.5).all()
    pts = np.concatenate([crowd[:30], spread, half, crowd[30:]]).astype(np.float32)
    bulk = Rig(0.5, 12)
    bulk.add(pts)
    dev = bulk.check()
    key = tuple(bulk.m.keys(crowd[:1])[0])
    assert len(dev[key]) == 60
    assert any(v[0] == 1 for v in dev) and any(v[0] == -1 for v in dev)        # +-0.25 * 2 = +-0.5 rounds away from zero
    ragged = Rig(0.5, 12)
    o, sizes = 0, [1, 7, 13, 100, 2, 64, 301]
    for b in range(len(pts)):
        if o >= len(pts):
            break
        c = sizes[b % len(sizes)]
        ragged.add(pts[o:o + c])
        o += c
    assert_same(ragged.check(), dev, False, "ragged vs bulk")      # (both in id order against the restatement above)


# ------------------------------------------------------------------ box delete
def test_box_delete_contents():
    """Tombstones leave the contents; the deleted and remaining counts equal the port's (ikd-Tree semantics), through a
    delete, the same delete again, and a re-insert into the deleted region."""
    from oracle import oracle as O
    rng = np.random.default_rng(5)
    pts = _cloud(rng, 3000, -8.0, 8.0)
    pts[:40] = np.float32([1.25, 1.25, 1.25]) + rng.uniform(-0.2, 0.2, (40, 3)).astype(np.float32)   # a crowded voxel, half in a box
    boxes = np.float32([[-2, -2, -2, 1.25, 1.3, 1.25], [4, -8, -8, 8, 8, 0]])
    rig = Rig(0.5, 14)
    rig.add(pts)
    port = O.OracleIvox(0.5, 18)
    port.add(np.c_[pts, np.zeros(len(pts), np.float32)], 0)
    n1 = rig.delete_boxes(boxes)
    assert n1 == port.delete_boxes(boxes) and n1 > 300
    assert rig.g.stats()["points"] == port.num_points
    assert rig.delete_boxes(boxes) == 0 == port.delete_boxes(boxes)
    more = _cloud(rng, 400, -2.0, 1.0)
    rig.add(more)
    port.add(np.c_[more, np.zeros(len(more), np.float32)], len(pts))
    assert rig.g.stats()["points"] == port.num_points


# ------------------------------------------------------------------ LRU, map level
def _out_and_back(rig, rng):
    xs = np.concatenate([np.arange(0, 80, 4.0), np.arange(80, -4, -8.0)])
    dist, prev = 0.0, xs[0]
    for x in xs:
        dist += abs(x - prev); prev = x
        n = int(rng.integers(100, 300))
        p = np.c_[x + rng.uniform(-6, 6, n), rng.uniform(-4, 4, n), rng.uniform(0, 1.5, n)].astype(np.float32)
        rig.add(p, dist)


def test_lru_out_and_back():
    rig = Rig(0.5, 14, capacity=300, max_distance=20.0)
    _out_and_back(rig, np.random.default_rng(3))
    assert rig.m.n["evicted"] > 1000 and rig.g.evict() == rig.m.n["evicted"], (rig.m.n, rig.g.evict())


def test_lru_recreated_voxel_keeps_all_its_points():
    """Capacity 10, max_distance 0: the oldest voxel is evicted by a new one and re-created by 20 points in the same batch."""
    rig = Rig(0.5, 12, capacity=10, max_distance=0.0)
    rig.add(np.c_[np.arange(11) * 2.0, np.zeros(11), np.zeros(11)], 0.0)
    rng = np.random.default_rng(2)
    b2 = np.r_[[[40.0, 0, 0]], rng.uniform(-0.2, 0.2, (20, 3))].astype(np.float32)
    rig.add(b2, 1.0)
    assert rig.m.n["recreated_over_8"] == 1 and rig.m.n["max_survivors"] == 20, rig.m.n
    st = rig.g.stats()
    assert (st["cells"], st["points"], st["dropped"]) == (10, 29, 0), st


def test_lru_voxel_evicted_and_recreated_repeatedly():
    """A voxel re-created in a batch is as young as the batch's distance, so it cannot be evicted again within the batch
    (max_distance >= 0): iVox evicts a voxel at most once per AddPoints call.  This drives many evictions and re-creations
    per batch (capacity 2) and pins that count."""
    rig = Rig(0.5, 12, capacity=2, max_distance=0.0)
    rng = np.random.default_rng(7)
    cells = np.float32([[0, 0, 0], [2, 0, 0], [4, 0, 0], [6, 0, 0]])
    for b in range(8):
        idx = rng.integers(0, 4, 40)
        rig.add(cells[idx] + rng.uniform(-0.2, 0.2, (40, 3)).astype(np.float32), float(b))
    assert rig.m.n["recreated"] > 10 and rig.m.n["evicted_twice"] == 0, rig.m.n


@pytest.mark.parametrize("capacity,max_distance", [(1, 0.0), (1, 2.5), (40, 0.0)])
def test_lru_small_capacity_and_zero_distance(capacity, max_distance):
    rig = Rig(0.5, 12, capacity=capacity, max_distance=max_distance)
    rng = np.random.default_rng(capacity + int(max_distance * 10))
    for b in range(10):
        rig.add(_cloud(rng, 60, -3.0, 3.0), float(b))
    assert rig.m.n["recreated"] > 0 and rig.m.n["evicted"] > 50, rig.m.n


def test_lru_across_table_rebuilds():
    """1024 lines: the retired lines cross half the table several times and the table is rebuilt (map_rehash) each time."""
    rig = Rig(0.5, 10, capacity=60, max_distance=1.0)
    rng = np.random.default_rng(9)
    for b in range(30):
        rig.add(np.c_[rng.uniform(b * 3, b * 3 + 8, 80), rng.uniform(-3, 3, 80), rng.uniform(0, 1, 80)].astype(np.float32), float(b * 3))
    assert rig.g.evict() > 1024 and rig.g.stats()["dropped"] == 0, (rig.g.evict(), rig.g.stats())


def test_lru_evicts_a_voxel_with_tombstones():
    """Box-deleted points of an evicted voxel were already taken off `points`: the eviction takes off the live ones only."""
    rig = Rig(0.5, 12, capacity=2, max_distance=0.0)
    a = np.float32([[0.1, 0.1, 0.1], [0.15, 0.1, 0.1], [0.2, 0.1, 0.1], [-0.1, 0.1, 0.1]])
    rig.add(np.r_[a, [[3, 0, 0], [6, 0, 0]]].astype(np.float32), 0.0)
    assert rig.delete_boxes(np.float32([[0.0, 0, 0, 1, 1, 1]])) == 3
    rig.add(np.float32([[9, 0, 0]]), 1.0)                 # evicts the voxel of `a`, its one live point with it
    assert rig.m.n["evicted"] == 1
    st = rig.g.stats()
    assert (st["cells"], st["points"]) == (3, 3), st


# ------------------------------------------------------------------ LRU through the LIO front-end
@pytest.mark.parametrize("reference_order,next_id", [(False, 0), (True, 0), (False, 2**31 - 5000)])
def test_lio_lru_contents_match_compiled_ivox(reference_order, next_id):
    """A drive through the block scene out and back over its own ground, with a small capacity and max_distance: voxels
    near the sensor are evicted and re-created by the scans that revisit them.  The compiled iVox is fed the two AddPoints
    calls of every scan (PointToAdd, then PointNoNeedDownsample, laserMapping.cpp:571-572), built from the tapped flags
    and world points at the tapped travel distance, and the contents must match after every scan."""
    import lsdreg
    from lsdreg import synth
    from oracle import eskf
    from oracle import oracle as O
    if not O.HAVE_REF_IVOX_DUMP:
        pytest.skip("oracle/_ref/libref_lio.so not built from this ref_lio.cpp (needs the reference at build time)")
    CAP, MAXD = 2500, 0.5
    g = lsdreg.LioFrontend(map_log2_lines=16)
    g.map.enable_lru(CAP, MAXD)
    g.set_reference_order(reference_order)
    g.set_next_id(next_id)
    res, max_points = float(g.params.ivox_resolution), int(g.params.max_points)
    r = O.RefIvox(res, 18, CAP, MAXD)
    m = IvoxRestated(res, CAP, MAXD)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    t0 = synth.block_center(0, 0) + np.array([1.0, -2.0, 0.0])
    steps = [0, 1, 2, 3, 4, 5, 4, 3, 2, 1, 0] if not EMU else [0, 1, 2, 1, 0]
    x = lsdreg.make_state(pos=t0, rot_xyzw=eskf.R_to_quat(Rgt))
    P = lsdreg.init_cov()
    nid = next_id
    for k, s in enumerate(steps):
        Rk = Rgt @ synth.rot_from_rpy(0, 0, 0.02 * s)
        tk = t0 + np.array([0.6 * s, 0.15 * s, 0.0])
        scan = synth.scan64(30 + k, 120 if EMU else 250, Rk, tk)
        P = P + np.eye(23) * 1e-2
        x, P, info = g.scan(scan, x, P)
        assert info["status"] in (lsdreg.OK, lsdreg.MAP_SEEDED), info
        flags, travel = g.get_map_flags()
        world = g.get_matches()["world"]
        n_bound = max(flags.shape[0], 1)          # a scan takes n_down ids (2 n_down in reference order, once registered)
        id_t2 = n_bound if (reference_order and info["status"] != lsdreg.MAP_SEEDED) else 0
        i = np.arange(flags.shape[0], dtype=np.int64)
        ids = ((nid + i + np.where(flags == 2, id_t2, 0) + 2**31) % 2**32 - 2**31).astype(np.int32)   # int32 wrap
        for f in (1, 2):
            sel = flags == f
            r.add_ids(world[sel], ids[sel], travel)
            m.add(world[sel], ids[sel], travel, batch_end=f == 2)
        nid = (nid + n_bound + id_t2) & 0x7fffffff
        dev = device_contents(g.map)
        ref = ref_contents(r)
        id_order = reference_order and next_id == 0
        assert_same(dev, ref, id_order, f"scan {k}: compiled iVox")
        assert ref == m.contents(), f"scan {k}: the restatement departs from the compiled iVox"
    assert m.n["evicted"] > 1000 and m.n["recreated"] > 0, m.n
    print("LIO LRU path counts", dict(m.n))
    if reference_order and next_id == 0:
        assert m.n["order_breaks"] == 0, m.n        # ids ascend in AddPoints order: choosing survivors by id would do
    elif not EMU:
        assert m.n["order_breaks"] > 0, m.n         # the drive re-creates voxels whose survivors an id threshold gets wrong
    if next_id != 0:
        assert (ids < 0).any() or nid < next_id         # the ids wrapped past 2^31 - 1 during the drive


# ------------------------------------------------------------------ documented deviations
def test_overfull_voxel_drops_exactly_the_excess():
    """More than 128 lines x 7 points in one voxel: `dropped` is the excess, the stored ids a subset of the inserted ones
    (which ones is atomic order, DESIGN §5e)."""
    rng = np.random.default_rng(4)
    n = 128 * 7 + 77
    g_pts = (np.float32([5.0, 5.0, 5.0]) + rng.uniform(-0.2, 0.2, (n, 3))).astype(np.float32)
    rig = Rig(0.5, 12, compiled=False)
    rig.g.insert(np.c_[g_pts, np.zeros(n, np.float32)], 0)
    st = rig.g.stats()
    assert (st["cells"], st["points"], st["dropped"]) == (1, 896, 77), st
    d = rig.g.dump()
    assert len(d["id"]) == 896 and len(set(d["id"].tolist())) == 896 and set(d["id"].tolist()) <= set(range(n))
    assert (d["voxel"] == [10, 10, 10]).all()
    assert not d["tombstone"].any()


def test_points_outside_the_key_range_are_dropped():
    lim = (1 << 18) * 0.5
    pts = np.float32([[lim * 1.01, 0, 0], [0, -lim * 1.01, 0], [0, 0, lim * 2], [1.0, 1.0, 1.0]])
    rig = Rig(0.5, 12, compiled=False)
    rig.g.insert(np.c_[pts, np.zeros(4, np.float32)], 0)
    st = rig.g.stats()
    assert (st["cells"], st["points"], st["dropped"]) == (1, 1, 3), st
    assert rig.g.dump()["id"].tolist() == [3]


def test_non_finite_points():
    """A NaN coordinate: the device's float -> int conversion gives 0, so the point is stored in voxel 0 along that axis
    (iVox would file it under INT_MIN; the SIMT emulator converts like x86 and drops it as out of range).  +-inf saturates and
    is dropped as out of range.  With the LRU on, the host mirror files the NaN point where the device did, so evicting
    that voxel later keeps cells and points consistent."""
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    pts = np.float32([[nan, 1.0, 1.0], [inf, 1.0, 1.0], [1.0, -inf, 1.0], [3.0, 3.0, 3.0]])
    rig = Rig(0.5, 12, capacity=1, max_distance=0.0, compiled=False)
    rig.g.insert(np.c_[pts, np.zeros(4, np.float32)], 0)
    st = rig.g.stats()
    d = rig.g.dump()
    if EMU:
        assert (st["cells"], st["points"], st["dropped"]) == (1, 1, 3), st
    else:
        assert (st["cells"], st["points"], st["dropped"]) == (2, 2, 2), st
        i = d["id"].tolist().index(0)
        assert tuple(d["voxel"][i]) == (0, 2, 2) and np.isnan(d["xyz"][i, 0]) and not d["tombstone"][i]
    rig.g.set_travel_distance(1.0)
    rig.g.insert(np.float32([[9.0, 9.0, 9.0, 0.0], [9.1, 9.0, 9.0, 0.0]]), 10)   # one eviction per point: both older voxels go
    st = rig.g.stats()
    assert (st["cells"], st["points"]) == (1, 2), st
    assert sorted(rig.g.dump()["id"].tolist()) == [10, 11]
