"""CPU: the voxel grid's leaf classes (one thread per small leaf, one warp per crowded one, one block per big one, the in-place
sort in global memory above the block's shared memory) at their boundaries, executed by the SIMT emulator (tests/simt) and compared bit for bit with the oracle."""
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)

_PROLOGUE = r'''
import sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + "/tests"); sys.path.insert(0, %(root)r + "/tests/simt")
import lsdreg, build_emu
lsdreg.capi.lib = lsdreg.capi.load_library(build_emu.build())
lsdreg.lib = lsdreg.capi.lib
'''


def test_voxelgrid_leaf_classes_under_the_simt_emulator():
    sys.path.insert(0, os.path.join(_HERE, "simt"))
    import build_emu
    build_emu.build()
    script = _PROLOGUE % {"root": _ROOT} + open(os.path.join(_HERE, "simt", "fuzz_vg_classes.py")).read()
    r = subprocess.run([sys.executable, "-c", script], cwd=_ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "FUZZ_VG_CLASSES_OK" in r.stdout, r.stdout[-3000:] + "\n" + r.stderr[-3000:]
