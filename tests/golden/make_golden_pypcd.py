"""Writes tests/golden/pypcd_keyframe.npz: what the PCD reader the reference vendors (third_party/pypcd.py) parses from the
cloud.pcd that lsd_keyframe_save writes for a seeded key frame, for tests/test_keyframe_io.py.  Needs the reference tree:

  python tests/golden/make_golden_pypcd.py <reference tree>

lzf (only needed for compressed files) is stubbed, and numpy 2 dropped the binary mode of np.fromstring the reader was written
against, so that one call is routed to np.frombuffer.
"""
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lsdreg  # noqa: E402
from test_keyframe_io import PYPCD_POINTS, PYPCD_SEED, _cloud  # noqa: E402

sys.modules.setdefault("lzf", types.ModuleType("lzf"))
sys.path.insert(0, os.path.join(sys.argv[1], "third_party"))
import pypcd  # noqa: E402

pts = _cloud(np.random.default_rng(PYPCD_SEED), PYPCD_POINTS)
with tempfile.TemporaryDirectory() as d:
    lsdreg.keyframe_save(d, 5, 1, pts, np.eye(4))
    pypcd.np.fromstring = lambda buf, dtype=float, **kw: np.frombuffer(buf, dtype=dtype)
    pc = pypcd.PointCloud.from_path(os.path.join(d, "cloud.pcd"))
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pypcd_keyframe.npz"),
                    fields=np.array(pc.fields), size=np.array(pc.size), type=np.array(pc.type), count=np.array(pc.count),
                    width=pc.width, height=pc.height, points=pc.points, data=pc.data,
                    x=np.asarray(pc.pc_data["x"]), z=np.asarray(pc.pc_data["z"]), intensity=np.asarray(pc.pc_data["intensity"]))
print("wrote pypcd_keyframe.npz:", pc.points, list(pc.fields), pc.data)
