"""GPU, whole sensor stream: the product (lsd_lio_scan) inside the reference's control flow, against the restated pipeline
(oracle/fastlio.py::OracleFastLio, itself pinned to the compiled reference to 1e-16 by tests/test_oracle_fastlio.py) —
IMU initialisation, the seeding scan, NEARBY74 -> NEARBY18, flg_EKF_inited, ten updates with map_incremental, WITH the
reference's stale Nearest_Points rows (lsd_lio_set_stale_rows).

The stale rows are the product's default since round 2.  Runs in a subprocess.
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

def run(stale, shape=0, ref_order=False):
    # ref_order: neighbours in the order IVox::GetClosestPoint returns them, on both sides; the oracle then IS the compiled
    # laserMapping.cpp to 2e-16 per scan (tests/test_oracle_fastlio.py), so the product is held to 1e-11 instead of 1e-6
    ext_R, ext_t = np.eye(3), np.zeros(3)
    orc = F.OracleFastLio(ext_R, ext_t, backend="port", stale_neighbours=stale, reference_order=ref_order)
    g = lsdreg.LioFrontend(map_log2_lines=18, ivox_nearby=lsdreg.STENCIL_NEARBY74)
    g.set_stale_rows(stale)
    g.set_reference_order(ref_order)
    tol = (1e-11, 1e-11, 1e-10) if ref_order else (1e-6, 1e-7, 1e-5)
    got = {}
    def product(und, x, P, nearby, ekf_inited):
        g.set_nearby(nearby); g.set_ekf_inited(ekf_inited)
        xs, Ps, info = g.scan(und, x.to_vec(), P)
        got.update(x=xs, P=Ps, info=info)
        return g.get_down()
    n_eff, updates, worst = [], 0, np.zeros(2)
    for f, frame in enumerate(T._stream(17, ext_R, ext_t)):
        T._feed(orc, *frame)
        got.clear()
        # teacher: the product's posterior, so both maps are grown from the same poses
        assert orc.step(teacher=(lambda: (E.State.from_vec(got["x"]), got["P"])), down_from=product)
        if not got:
            assert f < 6
            continue
        info = got["info"]
        if f == 6:
            assert info["status"] == lsdreg.MAP_SEEDED and g.map.stats()["cells"] == orc.lio.map.num_cells > 0
            continue
        updates += 1
        assert info["status"] == lsdreg.OK
        co = orc.counts()
        assert info["n_down"] == co["n_down"] and info["n_eff"] == co["n_eff"] and info["degenerate"] == co["degenerate"], (f, info, co)
        assert g.map.stats()["cells"] == orc.lio.map.num_cells, f
        xo, Po = orc.free_posterior
        d = np.abs(E.State.from_vec(got["x"]).boxminus(xo))
        worst = np.maximum(worst, [d[0:3].max(), d[3:6].max()])
        assert d[0:3].max() < tol[0] and d[3:6].max() < tol[1] and d.max() < tol[2], (f, d)   # bar: 1e-4 m / 1e-5 rad
        np.testing.assert_allclose(got["P"], Po, rtol=1e-6, atol=1e-12)
        n_eff.append(info["n_eff"])
    assert updates == 10
    assert g.reference_order_fallbacks() == 0
    print("stale", stale, "shape", shape, "ref_order", ref_order, "worst", worst, "n_eff", n_eff)
    return n_eff

a = run(True)
b = run(False)
run(True, ref_order=True)
# the stale rows matter on this stream: some update keeps effective points the plain search does not have
assert any(x > y for x, y in zip(a, b)) and all(x >= y - 2 for x, y in zip(a, b)), (a, b)
print("SEQUENCE_OK")
'''


def test_product_inside_the_reference_control_flow_with_stale_rows():
    r = subprocess.run([sys.executable, "-c", _SCRIPT % {"root": _ROOT}], cwd=_ROOT, capture_output=True, text=True, timeout=420)
    tail = (r.stdout[-3000:] + "\n" + r.stderr[-3000:])
    assert r.returncode == 0 and "SEQUENCE_OK" in r.stdout, tail
