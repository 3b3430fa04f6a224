"""GPU: floor detection (lsd_floor_*) against the restatement in tests/floor_oracle.py, stage by stage.

Every stage list (prefiltered, clipped, candidates, inliers) must be identical with order, the covariances bit for bit (which
pins the neighbour lists and their order), the normals within 1e-5, and the normal filter's decision identical for every point
whose restated |n_z| lies outside +-1e-5 of cos 20 deg.  RANSAC is compared on the device's own candidate cloud: draws,
flags, iterations, skipped, best model, coefficient bits and inliers."""
import math
import threading

import numpy as np
import pytest

import floor_oracle as FO
import lsdreg

pytestmark = pytest.mark.gpu

CLUTTER = FO.scene(6, n_ground=4000, ground_z=-0.3, radius=12.0, walls=6)
PRESETS = {"mapping": (lsdreg.FLOOR_MAPPING, -1.8), "ground": (lsdreg.FLOOR_GROUND, -0.3), "render": (lsdreg.FLOOR_RENDER, -0.3)}


@pytest.fixture(scope="module", autouse=True)
def _dev():
    lsdreg.init(0)


def _params(det: lsdreg.FloorDetector) -> dict:
    p = det.params
    return dict(prefilter_leaf=p.prefilter_leaf, distance_near=p.distance_near, distance_far=p.distance_far, clip_keep_d=p.clip_keep_d,
                clip_cut_d=p.clip_cut_d, use_normal_filtering=p.use_normal_filtering, normal_filter_deg=p.normal_filter_deg,
                viewpoint_z=p.viewpoint_z, ransac_threshold=p.ransac_threshold, ransac_probability=p.ransac_probability,
                ransac_max_iterations=p.ransac_max_iterations, floor_pts_thresh=p.floor_pts_thresh, floor_normal_deg=p.floor_normal_deg)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    """Bit-identical, except that any NaN equals any NaN (the device's quiet NaN has another payload than numpy's)."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(_bits(np.where(na, 0, a)), _bits(np.where(nb, 0, b)))


def check_against_restatement(det: lsdreg.FloorDetector, pts: np.ndarray, label: str = "") -> dict:
    res = det.detect(pts)
    p = _params(det)
    o = FO.detect(pts, p)
    assert np.array_equal(_bits(det.cloud("prefiltered")), _bits(o["prefiltered"])), label
    assert np.array_equal(_bits(det.cloud("clipped")), _bits(o["clipped"])), label
    assert res["n_clipped"] == o["clipped"].shape[0]
    cand = det.cloud("candidates")
    if p["use_normal_filtering"] and o["clipped"].shape[0]:
        nrm, cov6 = det.normals()
        assert _same(cov6, o["cov6"]), f"{label}: covariances differ"
        n_ok = np.isfinite(o["normals"][:, 0])
        assert np.array_equal(n_ok, np.isfinite(nrm[:, 0])), label
        d = np.minimum(np.abs(nrm[n_ok, :3] - o["normals"][n_ok, :3]).max(1), np.abs(nrm[n_ok, :3] + o["normals"][n_ok, :3]).max(1))
        assert d.max(initial=0.0) < 1e-5, f"{label}: normals differ by {d.max()}"
        cos20 = math.cos(p["normal_filter_deg"] * math.pi / 180.0)
        band = np.abs(o["abs_nz"].astype(np.float64) - cos20) <= 1e-5
        # the device's candidates are a subsequence of the (identical) clipped cloud: recover which points it kept
        keep_dev = np.zeros(o["clipped"].shape[0], bool)
        keep_o = np.zeros_like(keep_dev); keep_o[o["cand_idx"]] = True
        cb, clb = [r.tobytes() for r in _bits(cand)], [r.tobytes() for r in _bits(o["clipped"])]
        j = 0
        for i, row in enumerate(clb):
            if j < len(cb) and cb[j] == row:
                keep_dev[i] = True; j += 1
        assert j == len(cb), label
        print(f"{label}: {int(band.sum())} of {band.size} clipped points within 1e-5 of cos(20 deg)")
        assert np.array_equal(keep_dev[~band], keep_o[~band]), f"{label}: normal filter decisions differ"
        if band.any() and not np.array_equal(keep_dev, keep_o):
            return res   # an in-band decision differs: downstream stages are compared on the device's own cloud elsewhere
    assert np.array_equal(_bits(cand), _bits(o["candidates"])), label
    assert res["n_candidates"] == o["candidates"].shape[0]
    assert res["reason"] == o["reason"], (label, res["reason"], o["reason"])
    assert res["found"] == o["found"]
    if o["ransac"] is not None:
        check_ransac(det, res, cand, p, o["ransac"], label)
        if o["coeffs"] is not None:
            assert np.array_equal(_bits(res["coeffs"]), _bits(o["coeffs"])), (label, res["coeffs"], o["coeffs"])
    return res


def check_ransac(det, res, cand, p, rs, label=""):
    idx, flags, counts = det.samples()
    assert idx.shape[0] == rs["idx"].shape[0], (label, idx.shape[0], rs["idx"].shape[0])
    assert np.array_equal(flags, rs["flags"]), label
    good = flags >= 0
    assert np.array_equal(idx[good], rs["idx"][good]), label
    assert np.array_equal(counts, rs["counts"]), label
    assert (res["iterations"], res["skipped"], res["best_hypothesis"]) == (rs["iterations"], rs["skipped"], rs["best"]), label
    if rs["best"] >= 0:
        assert np.array_equal(_bits(det.cloud("inliers")), _bits(cand[rs["inliers"]])), label
        assert res["n_inliers"] == rs["inliers"].size


def test_ransac_on_the_device_candidates():
    det = lsdreg.FloorDetector(lsdreg.FLOOR_GROUND)
    pts = FO.scene(21, n_ground=20000, ground_z=-0.3, radius=15.0, walls=3, platform=6000)
    res = det.detect(pts)
    cand = det.cloud("candidates")
    rs = FO.ransac(cand, det.params.ransac_threshold)
    check_ransac(det, res, cand, _params(det), rs, "platform")
    assert res["found"]


@pytest.mark.parametrize("preset", sorted(PRESETS))
def test_end_to_end(preset):
    pid, gz = PRESETS[preset]
    det = lsdreg.FloorDetector(pid)
    cases = {
        "level": FO.scene(1, n_ground=30000, ground_z=gz, radius=20.0, walls=2),
        "roll4": FO.scene(2, n_ground=30000, ground_z=gz, roll_deg=4.0, radius=20.0, walls=2),
        "roll14": FO.scene(3, n_ground=30000, ground_z=gz, roll_deg=14.0, radius=20.0),
        "outside": FO.scene(4, n_ground=30000, ground_z=gz - 2.5, radius=20.0),
        "platform": FO.scene(5, n_ground=12000, ground_z=gz, radius=15.0, platform=10000),
    }
    want = {"level": FO.FOUND, "roll4": FO.FOUND, "roll14": FO.NOT_VERTICAL, "outside": FO.FEW_CANDIDATES}
    for name, pts in cases.items():
        res = check_against_restatement(det, pts, f"{preset}/{name}")
        if name in want:
            assert res["reason"] == want[name], (name, res["reason"])
        print(f"{preset}/{name}: reason={res['reason']} iterations={res['iterations']} batches={res['batches']} "
              f"launches={res['launches']} round_trips={res['round_trips']} coeffs={res['coeffs']}")


def test_multiple_batches_and_redraws():
    # walls kept (no normal filter): the best plane holds a fifth of the candidates, so RANSAC needs hundreds of draws
    det = lsdreg.FloorDetector(lsdreg.FLOOR_GROUND, use_normal_filtering=0, hypotheses_per_batch=16)
    res = check_against_restatement(det, CLUTTER, "clutter")
    assert res["batches"] > 1 and res["iterations"] > 16, res
    # duplicates: samples with a repeated point fail isSampleGood and are redrawn
    base = FO.scene(7, n_ground=1200, ground_z=-0.3, radius=8.0)
    dup = np.concatenate([base, base, base])
    res = check_against_restatement(lsdreg.FloorDetector(lsdreg.FLOOR_GROUND), dup, "duplicates")
    # exactly collinear candidates: 1000 redraws, no model
    k = np.arange(40, dtype=np.float32)
    line = np.stack([k / 8, k / 4, -k / 32, k], 1).astype(np.float32)
    det = lsdreg.FloorDetector(lsdreg.FLOOR_GROUND, use_normal_filtering=0, floor_pts_thresh=3)
    res = check_against_restatement(det, line, "collinear")
    assert res["reason"] == FO.NO_MODEL


def test_raw_scan_with_an_overfull_map_voxel():
    """100 k raw returns, one 0.5 m map voxel with 1500 points (a surface next to the sensor): the map drops points, every
    normal comes from the exact whole-cloud scan, and the covariances are still the restatement's bits."""
    rng = np.random.default_rng(8)
    pts = FO.scene(8, n_ground=98500, ground_z=-0.3, radius=30.0)
    blob = np.concatenate([rng.uniform([0.3, -0.2, -0.2], [0.7, 0.2, 0.2], (1500, 3)), rng.random((1500, 1))], 1).astype(np.float32)
    pts = np.concatenate([pts, blob])
    det = lsdreg.FloorDetector(lsdreg.FLOOR_GROUND)
    res = check_against_restatement(det, pts, "raw")
    assert res["map_dropped"] > 0 and res["found"]


def test_degenerate_inputs():
    det = lsdreg.FloorDetector(lsdreg.FLOOR_MAPPING)
    r = det.detect(np.zeros((0, 4), np.float32))
    assert r["reason"] == FO.EMPTY and not r["found"]
    r = check_against_restatement(det, np.array([[1, 0, -1.8, 0], [0, 1, -1.8, 0]], np.float32), "two points")
    assert r["reason"] == FO.FEW_CANDIDATES
    pts = FO.scene(9, n_ground=20000, ground_z=-1.8, radius=15.0)
    pts[::97, 0] = np.nan; pts[1::89, 1] = np.inf; pts[2::83, 2] = -np.inf
    for pid in (lsdreg.FLOOR_MAPPING, lsdreg.FLOOR_GROUND):
        q = pts.copy()
        if pid == lsdreg.FLOOR_GROUND:
            q[:, 2] += 1.5
        r = check_against_restatement(lsdreg.FloorDetector(pid), q, f"nonfinite/{pid}")
        assert r["found"]


def test_batch_size_changes_no_bit():
    pts = CLUTTER
    outs = []
    for B in (16, 256, 4096):
        det = lsdreg.FloorDetector(lsdreg.FLOOR_GROUND, use_normal_filtering=0, hypotheses_per_batch=B)
        r = det.detect(pts)
        idx, fl, cn = det.samples()
        outs.append((r, idx, fl, cn, det.cloud("inliers")))
    r0 = outs[0]
    assert r0[0]["iterations"] > 16
    for r in outs[1:]:
        for k in ("found", "reason", "iterations", "skipped", "best_hypothesis", "n_inliers", "n_candidates"):
            assert r[0][k] == r0[0][k], k
        assert np.array_equal(_bits(r[0]["coeffs"]), _bits(r0[0]["coeffs"]))
        for a, b in zip(r[1:4], r0[1:4]):
            assert np.array_equal(a, b)
        assert np.array_equal(_bits(r[4]), _bits(r0[4]))


def test_device_input_equals_host_input():
    import torch
    pts = FO.scene(12, n_ground=40000, ground_z=-1.8, radius=25.0, walls=2)
    det = lsdreg.FloorDetector(lsdreg.FLOOR_MAPPING)
    a = det.detect(pts)
    ia = det.cloud("inliers")
    b = det.detect(torch.from_numpy(pts).cuda())
    assert a["found"] and np.array_equal(_bits(a["coeffs"]), _bits(b["coeffs"]))
    assert np.array_equal(_bits(ia), _bits(det.cloud("inliers")))


def _lio_run(floor_thread: bool):
    from lsdreg import synth
    from oracle import eskf
    m = synth.block_map(1, 2, 2, 0.5)
    g = lsdreg.LioFrontend(map_log2_lines=20)
    g.map.insert(m, 0)
    g.set_next_id(m.shape[0])
    stop = threading.Event()
    n_frames = [0]

    def worker():
        det = lsdreg.FloorDetector(lsdreg.FLOOR_MAPPING)
        pts = FO.scene(13, n_ground=40000, ground_z=-1.8, radius=25.0, walls=2)
        while not stop.is_set():
            det.detect(pts)
            n_frames[0] += 1
    th = threading.Thread(target=worker) if floor_thread else None
    if th:
        th.start()
    xs = []
    P = lsdreg.init_cov()
    for s in range(3):
        Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3 + 0.02 * s)
        tgt = synth.block_center(0, 0) + np.array([1.0 + 0.3 * s, -2.0, 0.0])
        scan = synth.scan64(20 + s, 250, Rgt, tgt)
        prior = eskf.State()
        prior.rot = eskf.R_to_quat(Rgt)
        prior.pos = tgt
        x, P2, info = g.scan(scan, prior.to_vec(), P)
        xs.append(np.array(x))
    stop.set()
    if th:
        th.join()
        assert n_frames[0] > 0
    return np.stack(xs)


def test_concurrent_with_lio():
    a = _lio_run(False)
    b = _lio_run(True)
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
