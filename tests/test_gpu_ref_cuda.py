"""GPU pin of the NDT path against the COMPILED reference CUDA matcher (fast_gicp::NDTCuda / NDTCudaCore recompiled
for sm_90a: oracle/ref_cuda.cu -> oracle/_ref/libref_cuda.so).  Two properties of the reference bound how tightly it
can be matched: (1) its voxel hash accepts a table in which up to 1 % of the POINTS found no bucket within 10 probes and
silently drops their voxels (gaussian_voxelmap.cu:37-52,283-288) — which ones depends on the order of the atomics —
whereas this library (and the CPU restatement) keep every voxel; (2) it accumulates voxel moments with fp32 atomicAdd in
arbitrary order (:138-147).  Hence: its voxel set is a >= 98.5 % subset of ours, correspondence counts agree to 1 %,
costs and derivatives to 2 %, and the aligned pose to 5 mm."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HAVE = os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_cuda.so"))


@pytest.mark.skipif(not HAVE, reason="oracle/_ref/libref_cuda.so not built (needs /root/reference + nvcc)")
@pytest.mark.parametrize("neighbors", [7, 1])
def test_ndt_matches_compiled_reference_cuda(neighbors):
    import lsdreg
    from lsdreg import synth
    from oracle.reg import OracleMatcher, RefNdtCuda
    m = synth.block_map(1, 1, 1, 0.25)
    m[:, :2] -= np.array([60, 40], np.float32)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = np.array([1.0, -2.0, 1.8])
    scan = synth.scan64(2, 200, Rgt, tgt + np.array([60, 40, 0]))[::2].copy()
    dR, dt = synth.perturb(5, 0.5, 3.0)
    guess = np.eye(4); guess[:3, :3] = Rgt @ dR; guess[:3, 3] = tgt + dt
    Tgt = np.eye(4); Tgt[:3, :3] = Rgt; Tgt[:3, 3] = tgt
    g = lsdreg.Matcher("NDT_CUDA", ndt_neighbors=neighbors)
    o = OracleMatcher("ndt", neighbors=neighbors)
    r = RefNdtCuda(1.0, neighbors)
    for mm in (g, o, r):
        mm.set_target(m); mm.set_source(scan)
    assert g.stats()["n_voxels"] == o.n_voxels
    assert 0.985 * o.n_voxels <= r.n_voxels <= o.n_voxels
    for T in (guess, Tgt):
        er, Hr, br = r.linearize(T)
        eg, Hg, bg, ncg = g.cost(T)
        eo, Ho, bo = o.cost(T)
        assert ncg == o.n_corr and 0.985 * ncg <= r.n_corr <= ncg
        for e, H, b in ((eg, Hg, bg), (eo, Ho, bo)):
            np.testing.assert_allclose(e, er, rtol=2e-2)
            np.testing.assert_allclose(H, Hr, rtol=2e-2, atol=2e-2 * np.abs(Hr).max())
            np.testing.assert_allclose(b, br, rtol=2e-2, atol=5e-2 * np.abs(br).max())
    T2 = Tgt.copy(); T2[:3, 3] += [0.03, -0.02, 0.01]
    np.testing.assert_allclose(g.cost(T2, update=False, deriv=False)[0], r.compute_error(T2), rtol=2e-2)
    Tr = r.align(guess)
    Tg = g.align(guess)
    assert g.converged == r.converged
    assert np.abs(Tg[:3, 3] - Tr[:3, 3]).max() < 5e-3 and np.abs(Tg[:3, :3] - Tr[:3, :3]).max() < 1e-3


HAVE_VFE = os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_vfe.so"))


@pytest.mark.skipif(not HAVE_VFE, reason="oracle/_ref/libref_vfe.so not built (needs /root/reference + nvcc)")
@pytest.mark.parametrize("frames", [1, 4])
def test_voxelizer_matches_compiled_reference_kernels(frames):
    """lsd_vfe_* against the reference's own Preprocess / Voxelization kernels (recompiled for sm_90a).  The reference
    assigns voxel rows and point slots in atomic order, so the comparison is per voxel KEY: same window, same voxel set,
    and — for every voxel that holds no more points than the cap, where the reference is deterministic — the same fp16
    features up to the fp32 summation order (1 fp16 ulp)."""
    import lsdreg
    from oracle.vfe import RefVoxelizer
    import importlib.util
    spec = importlib.util.spec_from_file_location("_vfe_helpers", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_vfe.py"))
    helpers = importlib.util.module_from_spec(spec); spec.loader.exec_module(helpers)
    _frames = helpers._frames
    pts, motions = _frames(4)
    g = lsdreg.Voxelizer(max_frame_num=frames)
    r = RefVoxelizer(max_frame_num=frames)
    for f in range(4):
        tg = g.accumulate(pts[f], motions[f])
        tr = r.accumulate(pts[f], motions[f])
        assert tg == tr
        wg, wr = g.points(), r.points()
        np.testing.assert_allclose(wg, wr, rtol=2e-7, atol=1e-6)
        bit_equal = float((wg.view(np.int32) == wr.view(np.int32)).mean())
        assert bit_equal > 0.999, bit_equal                            # the motion-compensated window: same fp32 bits
        feat, idx, npts = g.voxelize(True)
        rf, ri = r.voxelize(True)
        assert feat.shape[0] == rf.shape[0] > 1000
        key = lambda a: (a[:, 1].astype(np.int64) << 40) | (a[:, 2].astype(np.int64) << 20) | a[:, 3].astype(np.int64)
        og, orr = np.argsort(key(idx)), np.argsort(key(ri))
        np.testing.assert_array_equal(idx[og], ri[orr])                 # identical voxel set
        small = npts[og] < 5                                            # below the cap: every point is in the mean on both sides
        a = feat[og][small].astype(np.float32); b = rf[orr][small].astype(np.float32)
        assert small.mean() > 0.5
        np.testing.assert_allclose(a, b, rtol=2e-3, atol=2e-3)
        assert float((feat[og][small].view(np.uint16) == rf[orr][small].view(np.uint16)).mean()) > 0.99
