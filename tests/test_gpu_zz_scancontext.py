"""GPU: ScanContext on the device (row N4, csrc/scancontext.cu) through the C ABI against the restatement
(oracle/scancontext.py, pinned bit-exact to the compiled reference by tests/test_oracle_scancontext.py) and the committed
golden vectors (tests/golden/scancontext_ref.npz, produced by the compiled reference).  Bars: descriptor bit-exact; keys
and pair distances bit-exact (same reduction order; 1e-12 would be the fallback bar if the device's atan / division ever
differed in the last bit, which would show up here as a flipped bin); shifts, candidate lists and matches identical.

The kernels' arithmetic (csrc/sc_math.h) is also pinned on the CPU (tests/sc_host_harness.cpp).  Runs in a
subprocess.
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
from oracle import scancontext as S
import test_oracle_scancontext as T

lsdreg.init(0)
clouds, n_places = T.sc_clouds()
sc = lsdreg.ScanContext(db_capacity=256, dist_thres=0.2)

# 1. descriptors + keys for all nine search offsets in one call
descs = []
for k, c in enumerate(clouds):
    d, rk, sk = sc.make(c, S.SEARCH_TRANS)
    for j, (dx, dy) in enumerate(S.SEARCH_TRANS):
        o = S.make(c, dx, dy)
        np.testing.assert_array_equal(d[j], o, err_msg=f"descriptor {k} offset {j}")
        np.testing.assert_array_equal(rk[j], S.ringkey(o)); np.testing.assert_array_equal(sk[j], S.sectorkey(o))
    descs.append(d[0].copy())
d, rk, sk = sc.make(np.zeros((0, 4), np.float32))
assert (d == 0).all() and (rk == 0).all()
print("make ok")

# 2. the golden vectors of the compiled reference
g = np.load(%(root)r + "/tests/golden/scancontext_ref.npz")
for k in range(g["clouds_n"].shape[0]):
    c = g["clouds"][k][: g["clouds_n"][k]]
    d, rk, sk = sc.make(c, g["offsets"][k][None, :])
    np.testing.assert_array_equal(d[0].reshape(-1), g["desc"][k]); np.testing.assert_array_equal(rk[0], g["ringkey"][k])
    np.testing.assert_array_equal(sk[0], g["sectorkey"][k])
dist, sh = sc.distance(g["desc"][g["pairs"][:, 0]], g["desc"][g["pairs"][:, 1]])
np.testing.assert_array_equal(sh, g["pair_shift"]); np.testing.assert_array_equal(dist, g["pair_dist"])
print("golden ok")

# 3. pair distances incl. an empty descriptor (no effective sector: 1e7, shift 0) and > 64 pairs (chunking)
rng = np.random.default_rng(3)
pairs = rng.integers(0, len(descs), (150, 2))
A = np.stack([descs[a] for a, _ in pairs] + [np.zeros((60, 20))]); B = np.stack([descs[b] for _, b in pairs] + [descs[0]])
dist, sh = sc.distance(A, B)
for i in range(A.shape[0]):
    od, os_ = S.distance(A[i], B[i])
    assert dist[i] == od and sh[i] == os_, (i, dist[i], od, sh[i], os_)
print("distance ok")

# 4. database + retrieval: empty database, fewer than 10 entries, the full one; both thresholds
assert sc.detect_closest(0) == (-1, 0.0, 1.0) and sc.detect_candidates(0) == []
for n_db in (3, n_places):
    for thres in (0.2, 0.6):
        sc.db_clear(); sc.dist_thres = thres
        sc.db_add(np.stack(descs[:n_db]))
        assert sc.db_size() == n_db
        db = S.Database(descs[:n_db], thres)
        hits = 0
        for qi, c in enumerate(clouds):
            dq, _, _ = sc.make(c, S.SEARCH_TRANS)
            idx, dist, sh, nc = sc.query(None, 9)
            for j in range(9):
                oc = db.candidates(dq[j])
                assert nc[j] == len(oc) == min(10, n_db)
                assert [(int(idx[j, t]), float(dist[j, t]), int(sh[j, t])) for t in range(nc[j])] == oc, (qi, j)
                assert sc.detect_closest(j) == db.detect_closest(dq[j]), (qi, j)
                assert sc.detect_candidates(j) == db.detect_candidates(dq[j]), (qi, j)
                hits += sc.detect_closest(j)[0] >= 0
            i2, d2, s2, n2 = sc.query(dq[:4])          # host descriptors in
            np.testing.assert_array_equal(i2, idx[:4]); np.testing.assert_array_equal(d2, dist[:4])
        print("retrieval ok", n_db, thres, "hits", hits)
# 5. database grown from made descriptors on the device == from host descriptors
sc.db_clear()
for c in clouds[:n_places]:
    sc.make(c); sc.db_add_made(0)
sc.make(clouds[-1], S.SEARCH_TRANS)
a = sc.query(None, 9)
sc.db_clear(); sc.db_add(np.stack(descs[:n_places])); sc.make(clouds[-1], S.SEARCH_TRANS)
b = sc.query(None, 9)
for x, y in zip(a, b):
    np.testing.assert_array_equal(x, y)
print("SC_OK")
'''


def test_scancontext_on_the_device_matches_the_restatement_and_the_golden_vectors():
    r = subprocess.run([sys.executable, "-c", _SCRIPT % {"root": _ROOT}], cwd=_ROOT, capture_output=True, text=True, timeout=420)
    tail = (r.stdout[-3000:] + "\n" + r.stderr[-3000:])
    assert r.returncode == 0 and "SC_OK" in r.stdout, tail
