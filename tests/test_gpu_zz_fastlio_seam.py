"""GPU: the LIO seam end to end (lsd_fastlio_* = fastlio_init / _imu_enqueue / _pcl_enqueue / fastlio_main / _odometry /
_state / _is_init on the device path) on a 17-frame synthetic sensor stream, free-running, against the restated pipeline
(oracle/fastlio.py::OracleFastLio, pinned to the compiled reference to 1e-12 per scan) and — when oracle/_ref travelled
with the snapshot — against the compiled reference pipeline itself.  Checked per frame: the same branch of fastlio_main
(first scan / IMU initialising / map seeded / update), is_init, feats_down_size; per update: pose within 1e-4 m / 1e-5 rad of
the restated pipeline STARTED FROM THE SAME PRIOR is covered by tests/test_gpu_zz_sequence.py (1e-16 there) — here all run
free, and this stream is chaotic (rounding differences grow about tenfold per scan early on, DESIGN.md section 4): the
restated pipeline itself ends 8e-4 m from the compiled reference after ten updates, the product (under the SIMT emulator)
3e-8 m from the restatement after the first update and 6e-4 m / 1.4e-3 m from restatement / reference after the tenth.  The
bar is therefore a plumbing bar: 5e-3 m / 1e-3 rad after ten updates, covariance within 15 % of sigma_i sigma_j.  fastlio_odometry / fastlio_state are checked against the filter state they are read from.

STATUS: written after this round's GPU budget was spent — never run on a GPU; the seam's host side IS covered on the CPU
(tests/test_fastlio_seam_host.py).  Runs in a subprocess.
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r'''
import sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests")
import numpy as np
import lsdreg
from oracle import eskf as E
from oracle import fastlio as F
import test_oracle_fastlio as T

lsdreg.init(0)
ext_R, ext_t = lsdreg.synth.rot_from_rpy(0.01, -0.02, 0.05), np.array([0.05, -0.02, 0.1])
g = lsdreg.FastLio(ext_R, ext_t, map_log2_lines=18)
o = F.OracleFastLio(ext_R, ext_t, backend="port", stale_neighbours=True)
ref = F.RefFastLio(ext_R, ext_t) if F.HAVE_REF_FASTLIO else None
updates, seeded, worst, worst_ref, prev_end = 0, 0, np.zeros(2), np.zeros(2), None
for f, frame in enumerate(T._stream(17, ext_R, ext_t)):
    for p in (g, o) + ((ref,) if ref else ()):
        T._feed(p, *frame)
    assert g.step() and o.step()
    if ref: assert ref.step()
    assert g.step() is False                      # one package per frame
    assert g.initialised == o.initialised, f
    last = g.last()
    co = o.counts()
    x, P = g.filter()
    s16, e16 = g.odometry(); st = g.state()
    xs = E.State.from_vec(x)
    np.testing.assert_allclose(e16[:3, 3], x[:3], atol=0, rtol=0)
    np.testing.assert_allclose(e16[:3, :3], E.quat_to_R(x[3:7] / np.linalg.norm(x[3:7])), atol=1e-15)
    if "iters" in o.last:                         # an iterated update ran
        updates += 1
        assert last["status"] == lsdreg.OK and abs(last["n_down"] - co["n_down"]) <= 2, (f, last, co)   # free-running: a point may cross a leaf border
        assert abs(last["n_eff"] - co["n_eff"]) <= max(3, co["n_eff"] // 200), (f, last, co)
        d = np.abs(xs.boxminus(o.state()[0]))
        worst = np.maximum(worst, [d[0:3].max(), d[3:6].max()])
        Po = o.state()[1]; sd = np.sqrt(np.abs(np.diag(Po)))
        assert (np.abs(P - Po) <= 0.15 * np.outer(sd, sd) + 1e-14).all(), f          # free-running: 15 %% of sigma_i sigma_j
        if ref:
            dr = np.abs(xs.boxminus(ref.state()[0]))
            worst_ref = np.maximum(worst_ref, [dr[0:3].max(), dr[3:6].max()])
            assert abs(last["n_down"] - ref.counts()["n_down"]) <= 2, f
        # the scan started where the previous one ended (contiguous scans: no prediction in between)
        if prev_end is not None:
            np.testing.assert_allclose(s16[:3, 3], prev_end[:3, 3], atol=1e-6)
        np.testing.assert_allclose(st[:3], s16[:3, 3], atol=0, rtol=0)
        assert abs(st[19] - 1.0) < 0.05           # mean_acc_norm: the platform starts at rest
        prev_end = e16
    else:
        seeded += last["status"] == lsdreg.MAP_SEEDED
        assert last["status"] in (lsdreg.OK, lsdreg.IMU_INITIALIZING, lsdreg.MAP_SEEDED), (f, last)
        assert updates == 0, f                    # once updates start, every frame updates
assert updates == 10 and seeded == 1, (updates, seeded)
print("worst vs restated", worst, "worst vs compiled reference", worst_ref)
assert worst[0] < 5e-3 and worst[1] < 1e-3, worst
if ref: assert worst_ref[0] < 5e-3 and worst_ref[1] < 1e-3, worst_ref
T._sane(E.State.from_vec(g.filter()[0]))
print("SEAM_OK")
'''


def test_the_lio_seam_end_to_end_against_the_restated_and_the_compiled_pipeline():
    r = subprocess.run([sys.executable, "-c", _SCRIPT % {"root": _ROOT}], cwd=_ROOT, capture_output=True, text=True, timeout=420)
    tail = (r.stdout[-3000:] + "\n" + r.stderr[-3000:])
    assert r.returncode == 0 and "SEAM_OK" in r.stdout, tail
