"""GPU: two launch-side changes that must not change a bit.  (1) Programmatic dependent launch (lsd_lio_set_pdl,
csrc/lsd_common.cuh) changes WHEN a kernel's blocks become resident, never what they compute; (2) the pipelined voxel grid
(lsd_lio_set_pipeline, csrc/lio.h) runs the downsample of a prefetched scan on the copy stream while the previous scan
iterates and hands its buffers to the scan that adopts it.  For both: a scan stream registered with the attribute on must give the same bits as with it off — state,
covariance, Nearest_Points ids, downsampled scan, map contents — with and without stale rows, and with the double-buffered
ingest (a copy-stream event between two PDL launches).

Both are ON by default since round 2; it stays as the bit-identity
guard of the default path against the plain-launch path.  Runs in a subprocess (its own CUDA context).
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import lsdreg
from lsdreg import synth
from oracle import eskf

lsdreg.init(0)
m = synth.block_map(1, 2, 2, 0.5)
steps = []
for s in range(6):
    Rgt = synth.rot_from_rpy(0.01 * s, -0.02, 0.3 + 0.05 * s)
    tgt = synth.block_center(0, 0) + np.array([1.0 + 0.4 * s, -2.0 + 0.1 * s, 0.0])
    scan = np.ascontiguousarray(synth.scan64(2 + s, 250 + 37 * (s %% 3), Rgt, tgt), np.float32)     # scans of different sizes: n_down changes from scan to scan
    dR, dt = synth.perturb(5 + s)
    prior = eskf.State(); prior.rot = eskf.R_to_quat(Rgt @ dR); prior.pos = tgt + dt
    steps.append((scan, prior.to_vec()))

class _Dev:
    """A device-resident scan for LioFrontend.scan / .prefetch: a CUDA torch tensor on a GPU; under the SIMT emulator
    ("device" memory is host memory) the numpy buffer itself, presented through the two attributes capi reads."""
    def __init__(self, a):
        self.a = a; self.shape = a.shape; self.is_cuda = True
    def data_ptr(self):
        return self.a.ctypes.data

def to_dev(scan):
    try:
        import torch
        if torch.cuda.is_available():
            return torch.from_numpy(scan).cuda()
    except Exception:
        pass
    return _Dev(scan)

def stream(shape, pdl, stale, prefetch, pipe=0, dev=False):
    f = lsdreg.LioFrontend(map_log2_lines=20, async_map_insert=1 if prefetch else 0)
    f.map.insert(m, 0); f.set_next_id(m.shape[0])
    f.set_knn_shape(shape); f.set_stale_rows(stale); f.set_pdl(pdl); f.set_pipeline(pipe)
    scans = [to_dev(sc) if dev else sc for sc, _ in steps]
    out = []
    for s, (scan, x0) in enumerate(steps):
        if prefetch and s + 1 < len(steps) and s != 3:      # scan 4 arrives unannounced: the voxel grid falls back to the main stream
            f.prefetch(scans[s + 1])
        x, P, info = f.scan(scans[s], x0, lsdreg.init_cov())
        mt = f.get_matches()
        out.append((x.copy(), P.copy(), f.get_down().copy(), mt["idx"].copy(), mt["cnt"].copy() if "cnt" in mt else None,
                    info["n_eff"], info["n_down"], info["iterations"]))
    st = f.map.stats()
    ps = f.pipeline_stats()
    assert ps == (dict(issued=4, adopted=4) if (pipe and prefetch) else dict(issued=0, adopted=0)), ps   # scans 1, 2, 3, 5 were announced
    f.close()
    return out, st

def same(a, sa, b, sb, what):
    assert sa == sb, (what, sa, sb)
    for s, (u, v) in enumerate(zip(a, b)):
        for j in range(4):
            np.testing.assert_array_equal(u[j].view(np.int64) if u[j].dtype == np.float64 else u[j].view(np.int32),
                                          v[j].view(np.int64) if v[j].dtype == np.float64 else v[j].view(np.int32),
                                          err_msg=f"{what} scan {s} field {j}")
        if u[4] is not None:
            np.testing.assert_array_equal(u[4], v[4])
        assert u[5:] == v[5:], (what, s, u[5:], v[5:])

# 1. programmatic dependent launch on / off
for shape, stale, prefetch in ((0, 0, 0), (0, 1, 1), (0, 0, 1), (0, 1, 0)):
    a, sa = stream(shape, 0, stale, prefetch)
    b, sb = stream(shape, 1, stale, prefetch)
    same(a, sa, b, sb, f"pdl: shape {shape} stale {stale} prefetch {prefetch}")
    print("pdl ok: shape", shape, "stale", stale, "prefetch", prefetch, "n_eff", [u[5] for u in a])

# 2. pipelined voxel grid (lsd_lio_set_pipeline): the prefetched scan is downsampled on the copy stream and adopted by buffer
#    swap; host scans and device-resident scans, with and without PDL, one scan of the stream arriving unannounced
base, sbase = stream(0, 0, 1, 0)
for pdl, dev in ((0, False), (1, False), (0, True), (1, True)):
    b, sb = stream(0, pdl, 1, 1, pipe=1, dev=dev)
    same(base, sbase, b, sb, f"pipeline: pdl {pdl} dev {dev}")
    print("pipeline ok: pdl", pdl, "device scans", dev)
b, sb = stream(0, 0, 1, 1, pipe=0, dev=True)      # announcing device scans without the pipeline is a no-op
same(base, sbase, b, sb, "prefetch_dev without pipeline")
print("PDL_OK")
'''


def test_pdl_stream_is_bit_identical_to_the_plain_launches():
    r = subprocess.run([sys.executable, "-c", _SCRIPT % {"root": _ROOT}], cwd=_ROOT, capture_output=True, text=True, timeout=420)
    tail = (r.stdout[-3000:] + "\n" + r.stderr[-3000:])
    assert r.returncode == 0 and "PDL_OK" in r.stdout, tail
