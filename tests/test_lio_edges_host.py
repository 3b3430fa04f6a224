"""CPU: the scene of tests/lio_edges.py reaches every edge class in the COMPILED reference's own outputs (ref_lio_hmodel,
ref_map_incremental and Eigen's QR, oracle/_ref), so that a class the GPU test counts cannot be empty unnoticed; and the
committed esti_plane fixture is what the compiled reference answers."""
import os

import numpy as np
import pytest

import lio_edges as L
from oracle import oracle as O

pytestmark = pytest.mark.skipif(not (O.HAVE_REF_IVOX_DUMP and hasattr(O.ref, "ref_esti_plane_qr")),
                                reason="oracle/_ref/libref_lio.so not built (needs the reference tree)")


@pytest.mark.parametrize("reference_order", [True, False])
def test_scene_reaches_every_class(reference_order):
    """reference_order=False drives the port (rows in ascending (d2, id) order), whose planes are Eigen's bit for bit."""
    scene = L.tuned_scene(reference_order)
    o = L.make_oracle(scene, reference_order)
    ev = L.oracle_eval(o, scene["scan1"], True)
    mi = L.oracle_map_incremental(o, scene["scan1"], True)
    counts = L.classes(scene, ev, mi)
    ev2 = L.oracle_eval(o, scene["scan2"], True)
    mi2 = L.oracle_map_incremental(o, scene["scan2"], True)
    counts.update(L.stale_classes(scene, ev2, mi2))
    print(counts)
    assert not [c for c, v in counts.items() if v == 0], counts
    lab = scene["label"]
    # what each label is there for
    for k in (1, 2, 3, 4):
        assert (ev["cnt"][lab == f"few_{k}"] == k).all()
    assert (ev["cnt"][lab == "empty"] == 0).all()
    assert (ev["selected"][lab == "body_zero"] == 0).all()
    assert (mi["flags"][np.char.startswith(lab.astype(str), "box_tie")] == 1).all()
    assert (mi["flags"][lab == "box_out"] == 2).all() and (mi["flags"][lab == "dist_tie"] == 1).all()
    assert (mi["flags"][lab == "dist_less"] == 0).all()
    st = np.isin(lab, ["stale_keep", "stale_drop"])
    assert (ev2["cnt"][st] == 5).all() and (ev2["idx"][st] == ev["idx"][st]).all()      # the rows of scan 1, kept


def test_committed_esti_plane_sets_are_the_compiled_references():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esti_plane_edges.npz"))
    pabcd, ok = O.ref_esti_plane(g["pts"], 0.1)
    qr = O.ref_esti_plane_qr(g["pts"])
    assert (pabcd.view(np.uint32) == g["pabcd"].view(np.uint32)).all() and (ok == g["ok"]).all()
    assert (qr["nonzero_pivots"] == g["nz"]).all() and (qr["perm"] == g["perm"]).all()
