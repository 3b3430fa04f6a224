"""GPU: the closure search of global alignment (lsd_galign_*).  Batched FAST_VGICP equals the single-pair kernels on the same
tables bit for bit (poses, flags, iterations, iteration logs, fitness) and takes as many rounds as its longest pair; a
search split into batches gives the bits of an unsplit one; cost and align agree with separate lsd_reg FAST_VGICP handles;
search() equals the restatement made of the reference's compiled SCManager and FastVGICP (tests/galign_oracle.py), finds
the planted overlaps and no closure for key frames in another block."""
import os

import numpy as np
import pytest

import galign_oracle as GO

pytestmark = pytest.mark.gpu

EMU = bool(os.environ.get("LSDREG_EMU"))          # SIMT emulator build: small clouds
N_AZ = (60, 90) if EMU else (200, 400)             # below / above the 16 384-point thread-shape switch on the GPU
BEAMS = 16 if EMU else 64


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


@pytest.fixture(scope="module")
def world():
    """Reference map: R key frames every 4 m on a line through block (0, 0).  New map: key frames 0.5 m beside every other
    reference key frame, turned by 1-2 rad (a second drive over the same road), then two in block (1, 0)."""
    from lsdreg import synth
    c0 = synth.block_center(0, 0)
    refs, ref_T, news, new_T, new_block, planted = [], [], [], [], [], []
    for i in range(6):
        R = synth.rot_from_rpy(0.0, 0.0, 0.3 * i)
        t = c0 + np.array([-10.0 + 4.0 * i, 2.0, 0.0])
        refs.append(synth.scan64(700 + i, N_AZ[i % 2], R, t, n_beams=BEAMS)); ref_T.append(_pose(R, t))
    for j, i in enumerate((0, 2, 3, 5)):
        R = synth.rot_from_rpy(0.0, 0.0, 0.3 * i + 1.0 + 0.3 * j)
        t = ref_T[i][:3, 3] + np.array([0.4, -0.3, 0.0])
        news.append(synth.scan64(800 + j, N_AZ[j % 2], R, t, n_beams=BEAMS)); new_T.append(_pose(R, t)); new_block.append(0)
        planted.append((j, i))
    c1 = synth.block_center(1, 0)
    for j in range(2):
        R = synth.rot_from_rpy(0.0, 0.0, 0.5 * j)
        t = c1 + np.array([5.0 * j - 3.0, -6.0, 0.0])
        news.append(synth.scan64(900 + j, N_AZ[j % 2], R, t, bi=1, n_beams=BEAMS)); new_T.append(_pose(R, t)); new_block.append(1)
    return dict(refs=refs, ref_T=np.array(ref_T), news=news, new_T=np.array(new_T), new_block=new_block, planted=planted)


def _aligner(world, **kw):
    import lsdreg
    ga = lsdreg.GlobalAligner(**kw)
    ref_slots = [ga.add_keyframe(c, True) for c in world["refs"]]
    new_slots = [ga.add_keyframe(c, False) for c in world["news"]]
    return ga, ref_slots, new_slots


@pytest.fixture(scope="module")
def aligner(world):
    return _aligner(world)


def _guesses(world, q, refs):
    """Guesses of new key frame q against reference key frames `refs`: the true relative pose perturbed by 0.3 m / 3 deg."""
    from lsdreg import synth
    out = []
    for k, i in enumerate(refs):
        T = np.linalg.inv(world["ref_T"][i]) @ world["new_T"][q]
        P = _pose(synth.rot_from_rpy(0.0, 0.0, np.deg2rad(3.0) * (-1) ** k), np.array([0.3, -0.2 * (-1) ** k, 0.0]))
        out.append(P @ T)
    return out


def test_batched_equals_serial(world, aligner):
    ga, ref_slots, new_slots = aligner
    for q in (0, 1):                                               # a new cloud below and one above the shape switch
        refs = [0, 1, 2, 3]
        G = _guesses(world, q, refs)
        far = np.eye(4); far[:3, 3] = [500.0, 500.0, 0.0]         # no correspondence anywhere
        spin = G[1].copy()                                         # 40 degrees off: a long or failed alignment
        spin[:3, :3] = GO.yaw2matrix(np.deg2rad(40.0))[:3, :3] @ spin[:3, :3]
        refs += [2, 1]; G += [far, spin.astype(np.float32).astype(np.float64)]
        slots = [ref_slots[i] for i in refs]
        b = ga.match(new_slots[q], slots, np.array(G))
        s = ga.match(new_slots[q], slots, np.array(G), serial=True)
        for k in ("final", "converged", "iterations", "fitness"):
            assert np.array_equal(b[k], s[k]), k
        for lb, ls in zip(b["iteration_logs"], s["iteration_logs"]):
            assert np.array_equal(lb, ls)
        assert not b["converged"][4] and b["converged"][:4].sum() >= 2
        evals = [ga.match(new_slots[q], [sl], np.array([g]), serial=True)["rounds"] for sl, g in zip(slots, G)]
        assert b["rounds"] == max(evals) < sum(evals) == s["rounds"]
        again = ga.match(new_slots[q], slots, np.array(G))         # tables built: one launch per round + one fitness launch
        assert again["launches"] == again["rounds"] + 1
        assert np.array_equal(again["final"], b["final"])
    sizes = {world["news"][q].shape[0] for q in (0, 1)}
    if not EMU:
        assert min(sizes) < 16384 <= max(sizes)


def test_cost_and_align_against_lsd_reg(world, aligner):
    """Separate lsd_reg FAST_VGICP handles: their voxel tables are accumulated in another order, so agreement to rounding."""
    import lsdreg
    ga, ref_slots, new_slots = aligner
    q, refs = 1, [2, 3]
    G = _guesses(world, q, refs)
    m = ga.match(new_slots[q], [ref_slots[i] for i in refs], np.array(G))
    for k, i in enumerate(refs):
        r = lsdreg.Matcher("FAST_VGICP")
        r.set_target(world["refs"][i]); r.set_source(world["news"][q])
        for T in (G[k], m["final"][k]):
            e, H, b, n = ga.cost(new_slots[q], ref_slots[i], T)
            e2, H2, b2, n2 = r.cost(T)
            assert n == n2
            np.testing.assert_allclose(e, e2, rtol=1e-12)
            np.testing.assert_allclose(H, H2, rtol=1e-12, atol=1e-12 * np.abs(H2).max())
            np.testing.assert_allclose(b, b2, rtol=1e-12, atol=1e-12 * np.abs(b2).max())
            e3 = ga.cost(new_slots[q], ref_slots[i], T, update=False, deriv=False)[0]
            np.testing.assert_allclose(e3, r.cost(T, update=False, deriv=False)[0], rtol=1e-12)
        r.align(G[k].astype(np.float32))
        T2, _ = r.final()
        assert bool(m["converged"][k]) == r.converged
        assert np.abs(m["final"][k][:3, 3] - T2[:3, 3]).max() < 1e-6
        D = m["final"][k][:3, :3].T @ T2[:3, :3]
        assert np.linalg.norm(D - D.T) / (2 * np.sqrt(2)) < 1e-7
        r.close()


def test_chunked_search_equals_unchunked(world, aligner):
    """One search over all new key frames (one batch) and one search per new key frame (a batch each), on the same tables."""
    ga, ref_slots, new_slots = aligner
    full = ga.search(new_slots)
    fm = ga.matches()
    assert ga.stats()["batches"] == 1
    part, pm = [], []
    for s in new_slots:
        part += ga.search([s])
        pm += ga.matches()
    assert len(full) == len(part) and len(fm) == len(pm) and len(fm) > len(full) > 0
    for a, b in zip(full, part):
        assert (a["ref_slot"], a["new_slot"]) == (b["ref_slot"], b["new_slot"])
        assert np.array_equal(a["relpose"], b["relpose"]) and a["score"] == b["score"]
    for a, b in zip(fm, pm):
        assert a == b
    # one search split by the memory budget: batches of whole new key frames, the same bits
    ga.set_max_batch_points(1)
    try:
        split = ga.search(new_slots)
        sm = ga.matches()
        assert ga.stats()["batches"] > 1   # one per new key frame with matches (those without any cost nothing)
    finally:
        ga.set_max_batch_points(1 << 24)
    assert sm == fm and len(split) == len(full)
    for a, b in zip(full, split):
        assert (a["ref_slot"], a["new_slot"]) == (b["ref_slot"], b["new_slot"])
        assert np.array_equal(a["relpose"], b["relpose"]) and a["score"] == b["score"]


@pytest.mark.skipif(not GO.HAVE_REF, reason="oracle/_ref (compiled reference SCManager / FastVGICP) not built")
def test_search_matches_oracle_and_finds_overlaps(world, aligner):
    ga, ref_slots, new_slots = aligner
    closures = ga.search(new_slots)
    tried = ga.matches()
    o = GO.OracleGlobalAlignment(world["refs"])
    oc, ot = o.search(world["news"])
    slot_of_ref = {s: i for i, s in enumerate(ref_slots)}
    slot_of_new = {s: q for q, s in enumerate(new_slots)}
    # match lists: index, sc_dist, sc_yaw identical, in the same order
    assert [(slot_of_new[m["new_slot"]], slot_of_ref[m["ref_slot"]], m["sc_dist"], m["sc_yaw"]) for m in tried] == \
        [(r["new"], r["ref"], float(r["sc_dist"]), float(r["sc_yaw"])) for r in ot]
    assert [m["converged"] for m in tried] == [r["converged"] for r in ot]
    # closures: same set, order, poses and scores
    assert [(slot_of_new[c["new_slot"]], slot_of_ref[c["ref_slot"]]) for c in closures] == [(r["new"], r["ref"]) for r in oc]
    # Poses and scores to 1e-4 m / 1e-5 rad / 1e-5 relative.  The one allowance: a pair whose outcome changes between builds
    # of its reference key frame's target tables on the GPU (measured here on three more handles) is held to twice that
    # spread instead, since the reference cannot be matched more closely than the product matches itself.  Such a pair
    # must be rare: at most one in this scene (new 3 / reference 5, whose target build lsd_reg FAST_VGICP handles do not
    # reproduce either; DESIGN.md section 5e).
    others = []
    for _ in range(3):
        g2, _, ns2 = _aligner(world)
        others.append(g2.search(ns2))
        g2.close()
    sensitive = 0
    for k, (c, r) in enumerate(zip(closures, oc)):
        builds = [c] + [o2[k] for o2 in others]
        assert all((b["ref_slot"], b["new_slot"]) == (c["ref_slot"], c["new_slot"]) for b in builds)
        dt = float(np.abs(c["relpose"][:3, 3] - r["relpose"][:3, 3]).max())
        dr = _rot_err(c["relpose"], r["relpose"])
        ds = abs(c["score"] - r["score"]) / abs(r["score"])
        st = max(float(np.abs(b["relpose"][:3, 3] - c["relpose"][:3, 3]).max()) for b in builds)
        sr = max(_rot_err(b["relpose"], c["relpose"]) for b in builds)
        ss = max(abs(b["score"] - c["score"]) / abs(c["score"]) for b in builds)
        sensitive += st > 0
        assert dt < max(1e-4, 2 * st) and dr < max(1e-5, 2 * sr) and ds < max(1e-5, 2 * ss), (k, dt, dr, ds, st, sr, ss)
    assert sensitive <= 1
    # the planted overlaps: every one a closure, within 5 cm of T_ref^-1 T_new; nothing from the other block
    got = {(slot_of_new[c["new_slot"]], slot_of_ref[c["ref_slot"]]): c for c in closures}
    for q, i in world["planted"]:
        assert (q, i) in got, (q, i)
        Tt = np.linalg.inv(world["ref_T"][i]) @ world["new_T"][q]
        assert np.abs(got[(q, i)]["relpose"][:3, 3] - Tt[:3, 3]).max() < 0.05
    assert all(world["new_block"][q] == 0 for q, _ in got)
    assert all(m["accepted"] == (m["converged"] and m["score"] < 1.5) for m in tried)


def _rot_err(Ta, Tb):
    D = Ta[:3, :3].astype(np.float64).T @ Tb[:3, :3].astype(np.float64)
    return float(np.linalg.norm(D - D.T) / (2 * np.sqrt(2)))
