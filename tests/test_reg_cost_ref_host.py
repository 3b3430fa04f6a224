"""CPU pin of the cost restatement (reg_cost_ref.py) against the C oracle (oracle/lsd_oracle.c), which test_oracle_reg.py
pins to the compiled FastGICP / FastVGICP.  The restatement is fed the oracle's own normals and voxel tables; the oracle adds
the same terms in its own order, so each of its 28 sums must lie within gamma(m - 1) * sum |t| of the exact sum of the
restated terms.  The restatement is also held to the independent float64 statement of the mathematics."""
import numpy as np
import pytest

import reg_build_ref as RB
import reg_cost_ref as RC


@pytest.fixture(scope="module")
def scene():
    """test_oracle_reg.py's scene: a block map cropped to 60 m x 60 m and a near-range scan."""
    from lsdreg import synth
    crop = lambda m: m[(np.abs(m[:, 0]) < 30) & (np.abs(m[:, 1]) < 30)].copy()
    m = synth.block_map(1, 1, 1, 0.5)
    m[:, :2] -= np.array([60, 40], np.float32)
    dense = synth.block_map(1, 1, 1, 0.25)                               # NDT: voxels of more than 6 points
    dense[:, :2] -= np.array([60, 40], np.float32)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = np.array([1.0, -2.0, 1.8])
    scan = synth.scan64(2, 200, Rgt, tgt + np.array([60, 40, 0]))
    scan = scan[np.linalg.norm(scan[:, :3], axis=1) < 25][::2].copy()
    dR, dt = synth.perturb(5, 0.3, 2.0)
    guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
    Tgt = np.eye(4); Tgt[:3, :3] = Rgt; Tgt[:3, 3] = tgt
    T2 = Tgt.copy(); T2[:3, 3] += [0.03, -0.02, 0.01]
    return dict(tgt=crop(m), dense=crop(dense), src=scan, guess=guess, Tgt=Tgt, T2=T2)


def _oracle_ndt_table(o, pts):
    from oracle import oracle as O
    coords = np.array(sorted(RB.ndt_table(pts, o.res)), np.int64)
    count = np.zeros(len(coords), np.int64)
    mean, second = np.zeros((len(coords), 3)), np.zeros((len(coords), 6))
    mo, no = np.zeros(3, np.float32), np.zeros(3, np.float32)
    for k, c in enumerate(coords):
        count[k] = O.port.orc_ndt_voxel(o.ndt, *(int(v) for v in c), mo, no)
        mean[k], second[k, :3] = mo, no
    assert count.min() > 0 and len(coords) == o.n_voxels
    return dict(coord=coords, count=count, mean=mean, second=second)


def _check(dev, terms, deriv):
    e, H, b = dev
    return RC.check_sums(RC.unpack(e, H.reshape(6, 6), b), terms.flat(), deriv)


@pytest.mark.parametrize("n_off", [1, 7, 27])
def test_ndt_restatement_matches_oracle(scene, n_off):
    from oracle.reg import OracleMatcher
    o = OracleMatcher("ndt", neighbors=n_off)
    o.set_target(scene["dense"]); o.set_source(scene["src"])
    tab = RC.Table(_oracle_ndt_table(o, o.tgt))
    for T in (scene["guess"], scene["Tgt"]):
        t = RC.ndt_terms(o.src, tab, o.res, n_off, T, T)
        dev = o.cost(T)
        assert o.n_corr == t.n_corr and t.used.sum() > 1000
        _check(dev, t, True)
        RC.math_check_ndt(T, o.src, t)
    for deriv in (True, False):           # update = False: looked up at Tgt (the last linearisation), evaluated at T2
        t = RC.ndt_terms(o.src, tab, o.res, n_off, scene["Tgt"], scene["T2"], deriv)
        _check(o.cost(scene["T2"], update=False, deriv=deriv), t, deriv)
        RC.math_check_ndt(scene["T2"], o.src, t)


def test_gicp_restatement_matches_oracle(scene):
    from oracle.reg import OracleMatcher
    o = OracleMatcher("gicp")
    o.set_target(scene["tgt"]); o.set_source(scene["src"])
    for T in (scene["guess"], scene["Tgt"]):
        corr, _ = RC.gicp_nn(o.src, o.tgt, T, o.max_corr)
        dev = o.cost(T)
        np.testing.assert_array_equal(corr, o.corr)
        t = RC.gicp_terms(o.src, o.tgt, o.src_nrm, o.tgt_nrm, corr, T, T)
        assert t.n_corr > 1000
        _check(dev, t, True)
        RC.math_check_gicp(t, o.src_nrm, o.tgt_nrm, T)
    for deriv in (True, False):
        t = RC.gicp_terms(o.src, o.tgt, o.src_nrm, o.tgt_nrm, corr, scene["Tgt"], scene["T2"], deriv)
        _check(o.cost(scene["T2"], update=False, deriv=deriv), t, deriv)
        RC.math_check_gicp(t, o.src_nrm, o.tgt_nrm, scene["Tgt"])


def _floors(seed, n, z_levels, half=6.0):
    """Horizontal patches at heights that are exact in float (sums of up to 20 of them stay exact): every k-NN covariance
    then has an exact zero z row, its normal is +-e_z exactly and every 0.999 n_a n_b is symmetric in (a, b)."""
    rng = np.random.default_rng(seed)
    parts = [np.concatenate([rng.uniform(-half, half, (n, 2)), np.full((n, 1), z)], 1) for z in z_levels]
    P = np.concatenate(parts).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([P, np.zeros((P.shape[0], 1), np.float32)], 1))


@pytest.mark.parametrize("n_off", [1, 7, 27])
def test_vgicp_restatement_matches_oracle(n_off):
    """The oracle accumulates its voxel covariances as full 3x3 sums, (0.999 n_a) n_b and (0.999 n_b) n_a apart, and
    inverts the full matrix; the kernel reads the upper triangle.  On a scene whose normals are +-e_z and whose poses
    rotate about z only, both triangles are the same numbers and the chain is exact to the reduction bound."""
    from lsdreg import synth
    from oracle import oracle as O
    from oracle.reg import OracleMatcher
    tgt = _floors(1, 3000, [-3.0, 0.25, 3.5])
    src = _floors(2, 800, [-3.0, 0.25, 3.5], half=5.0)
    o = OracleMatcher("vgicp", neighbors=n_off)
    o.set_target(tgt); o.set_source(src)
    assert np.all(np.abs(o.tgt_nrm[:, :2]) == 0) and np.all(np.abs(o.src_nrm[:, :2]) == 0)
    ref = RB.vgicp_table(tgt, o.tgt_nrm)
    coords = np.array(sorted(ref), np.int64)
    count = np.zeros(len(coords), np.int64)
    mean, second = np.zeros((len(coords), 3)), np.zeros((len(coords), 6))
    mo, co = np.zeros(3), np.zeros(9)
    for k, c in enumerate(coords):
        count[k] = O.port.orc_vgicp_voxel(o.vg, *(int(v) for v in c), mo, co)
        assert np.array_equal(co.reshape(3, 3), co.reshape(3, 3).T)
        mean[k], second[k] = mo, co[[0, 1, 2, 4, 5, 8]]
    assert count.min() > 0 and len(coords) == o.n_voxels
    tab = RC.Table(dict(coord=coords, count=count, mean=mean, second=second))
    T = np.eye(4); T[:3, :3] = synth.rot_from_rpy(0.0, 0.0, 0.2); T[:3, 3] = [0.3, -0.2, 0.05]
    T2 = T.copy(); T2[:3, 3] += [0.02, 0.01, -0.03]
    t = RC.vgicp_terms(o.src, o.src_nrm, tab, o.res, n_off, T, T)
    dev = o.cost(T)
    assert o.n_corr == t.n_corr and t.n_corr > 500
    _check(dev, t, True)
    RC.math_check_vgicp(t, o.src, o.src_nrm, T)
    for deriv in (True, False):
        t = RC.vgicp_terms(o.src, o.src_nrm, tab, o.res, n_off, T, T2, deriv)
        _check(o.cost(T2, update=False, deriv=deriv), t, deriv)
        RC.math_check_vgicp(t, o.src, o.src_nrm, T)
